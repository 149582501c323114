// esm_b200 — C ABI (include/esmb200.h): host-side orchestration of the sm_90a kernels.
//
// Everything here is plain C-callable: device pointers in, launches on the caller's stream, no torch types.
// Host work per call is limited to encoding a handful of TMA descriptors (cuTensorMapEncodeTiled) and
// launching 7 kernels per TransformerLayer:
//   LN1->fp16 | QKV GEMM (+bias, q scale, RoPE) | attention | out-proj GEMM (+bias, residual)
//   LN2->fp16 | fc1 GEMM (+bias, erf-GELU)      | fc2 GEMM (+bias, residual)
#include "../../include/esmb200.h"

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include <mutex>

#include "align.cuh"
#include "attention8.cuh"
#include "attention_contact.cuh"
#include "attention_probs.cuh"
#include "common.cuh"
#include "elementwise.cuh"
#include "gemm2.cuh"
#include "gemm_fp8.cuh"
#include "jacobian.cuh"
#include "knn.cuh"
#include "msa_select.cuh"
#include "sampling.cuh"
#include "tied_attention.cuh"

using namespace esmb200;

namespace {

thread_local std::string g_last_error;

int fail(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

int fail_cuda(cudaError_t e, const char* what) {
  if (e == cudaErrorMemoryAllocation)
    return fail(ESMB200_ENOMEM, std::string("CUDA out of memory. (") + what + ")");
  return fail(ESMB200_ECUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

#define CK(expr)                                        \
  do {                                                  \
    cudaError_t _e = (expr);                            \
    if (_e != cudaSuccess) return fail_cuda(_e, #expr); \
  } while (0)


// ---- launch accounting + optional per-launch CUDA-event timing (bench.py's roofline numbers) --------------------
enum ProfTag : int { T_LN1 = 0, T_QKV, T_ATTN, T_OUT, T_LN2, T_FC1, T_FC2, T_KEYBITS, T_EMBED, T_LN_F32, T_PROBS,
                     T_CONVERT, T_GEMM_OTHER, T_MEANPOOL, T_TIED_SCORES, T_TIED_SOFTMAX, T_TIED_PV, T_LOG_SOFTMAX,
                     T_WINDOW_MERGE, T_JACOBIAN, T_SAMPLING, T_MSA_SELECT, T_KNN, T_ALIGN, T_COUNT };
struct Profiler {  // process-wide, guarded by `mu`: launches may come from several host threads / streams
  std::mutex mu;
  bool on = false;
  std::vector<cudaEvent_t> ev;  // pairs (start, stop)
  std::vector<int> tag;
  size_t used = 0;              // events used
  long long launches = 0;       // kernels launched by this library since load
};
Profiler g_prof;

struct ProfScope {
  cudaStream_t st;
  bool rec;
  size_t slot = 0;
  ProfScope(int tag, cudaStream_t s) : st(s), rec(false) {
    std::lock_guard<std::mutex> lk(g_prof.mu);
    ++g_prof.launches;
    if (g_prof.on && g_prof.used + 2 <= g_prof.ev.size()) {
      rec = true;
      slot = g_prof.used;
      g_prof.used += 2;
      g_prof.tag.push_back(tag);
      cudaEventRecord(g_prof.ev[slot], st);
    }
  }
  ~ProfScope() {
    if (rec) cudaEventRecord(g_prof.ev[slot + 1], st);
  }
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// 2D row-major [rows, cols] (cols contiguous) of e4m3 (esize 1), fp16 (esize 2) or fp32 (esize 4);
// box = {128 bytes of columns, box_rows}, 128B swizzle.
int make_tmap_2d(CUtensorMap* map, const void* ptr, int esize, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                 uint32_t box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) return fail(ESMB200_ECUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld_elems * esize) % 16 != 0)
    return fail(ESMB200_EINVAL, "TMA operand must be 16-byte aligned with a 16-byte multiple row pitch");
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld_elems * (uint64_t)esize};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esize), box_rows};
  cuuint32_t estr[2] = {1, 1};
  const CUtensorMapDataType dt = esize == 1   ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                 : esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16
                                              : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = enc(map, dt, 2,
                   const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[160];
    snprintf(buf, sizeof buf, "cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu ld=%llu box_rows=%u", (int)r,
             (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)ld_elems, box_rows);
    return fail(ESMB200_ECUDA, buf);
  }
  return ESMB200_OK;
}

int make_tmap_f16(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld_elems,
                  uint32_t box_rows) {
  return make_tmap_2d(map, ptr, 2, rows, cols, ld_elems, box_rows);
}

// output of gemm2_f16_kernel: dense row-major [rows, cols] fp16 (esize 2) or fp32 (esize 4), written in boxes of one
// MMA warpgroup's 64 rows
int make_gemm_out_map(CUtensorMap* map, const void* out, int esize, uint64_t rows, uint64_t cols) {
  return make_tmap_2d(map, out, esize, rows, cols, cols, gemm2_cfg::OUT_BOX_ROWS);
}

// 64-wide column slots per head on the attention side: 1 for head_dim <= 64, 2 up to 128 (elementwise.cuh head_slot)
inline int head_slots(int E, int H) { return (H > 0 && E / H > 64) ? 2 : 1; }

constexpr int kMaxDevices = 64;

int num_sms() {  // per device: one process may drive several GPUs
  static int n[kMaxDevices] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= kMaxDevices) dev = 0;
  if (n[dev] == 0) cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
  return n[dev];
}

int check_device() {
  static int ok[kMaxDevices] = {};  // 0 unknown, 1 sm_90, -1 other
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return fail(ESMB200_ECUDA, "no CUDA device");
  if (dev < 0 || dev >= kMaxDevices) return fail(ESMB200_ECUDA, "device ordinal out of range");
  if (ok[dev] == 0) {
    int major = 0;
    cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
    ok[dev] = (major == 9) ? 1 : -1;
  }
  if (ok[dev] < 0)
    return fail(ESMB200_ECUDA, "esmb200 requires an sm_90a (Hopper H100) device; there is no fallback path");
  return ESMB200_OK;
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// esmb200_contact_accumulate's limit (its shared memory holds 8 rows of S floats)
constexpr int kContactMaxS = 1024;
const char* const kContactMaxSMsg = "contact head supports at most 1024 positions";

template <bool SPLIT>
cudaError_t launch_gemm_epi(int epi, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to,
                            const GemmParams& p, cudaStream_t st) {
  switch (epi) {
    case EPI_QKV_ROPE: return launch_gemm2_epi<EPI_QKV_ROPE, SPLIT>(ta, tb, to, p, num_sms(), st);
    case EPI_BIAS_RESIDUAL: return launch_gemm2_epi<EPI_BIAS_RESIDUAL, SPLIT>(ta, tb, to, p, num_sms(), st);
    case EPI_BIAS_GELU: return launch_gemm2_epi<EPI_BIAS_GELU, SPLIT>(ta, tb, to, p, num_sms(), st);
    case EPI_BIAS_F32: return launch_gemm2_epi<EPI_BIAS_F32, SPLIT>(ta, tb, to, p, num_sms(), st);
    case EPI_BIAS_GELU_F32: return launch_gemm2_epi<EPI_BIAS_GELU_F32, SPLIT>(ta, tb, to, p, num_sms(), st);
    default: return cudaErrorInvalidValue;  // launch_gemm rejects unknown epilogues first
  }
}

int launch_gemm(int epi, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const GemmParams& p,
                cudaStream_t st, int tag = T_GEMM_OTHER, bool split = false) {
  ProfScope ps(tag, st);
  // fp32x3 precision: operands stored as fp16 hi | lo along K (gemm2.cuh)
  if (split && p.K % 64 != 0) return fail(ESMB200_EINVAL, "fp32x3 precision needs K % 64 == 0");
  if (epi < EPI_QKV_ROPE || epi > EPI_BIAS_GELU_F32) return fail(ESMB200_EINVAL, "unknown GEMM epilogue");
  const cudaError_t e =
      split ? launch_gemm_epi<true>(epi, ta, tb, to, p, st) : launch_gemm_epi<false>(epi, ta, tb, to, p, st);
  if (e != cudaSuccess) return fail_cuda(e, split ? "gemm launch (fp32x3)" : "gemm launch");
  return ESMB200_OK;
}

// fp8 precision (gemm_fp8.cuh): epilogues EPI_QKV_ROPE (fp16 out), EPI_BIAS_RESIDUAL (fp32 x += y), EPI_GELU_FP8 (e4m3
// out + scales)
int launch_gemm_fp8(int epi, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const Fp8GemmParams& p,
                    cudaStream_t st, int tag = T_GEMM_OTHER) {
  ProfScope ps(tag, st);
  cudaError_t e;
  switch (epi) {
    case EPI_QKV_ROPE: e = launch_gemm_fp8_epi<EPI_QKV_ROPE>(ta, tb, to, p, num_sms(), st); break;
    case EPI_BIAS_RESIDUAL: e = launch_gemm_fp8_epi<EPI_BIAS_RESIDUAL>(ta, tb, to, p, num_sms(), st); break;
    case EPI_GELU_FP8: e = launch_gemm_fp8_epi<EPI_GELU_FP8>(ta, tb, to, p, num_sms(), st); break;
    default: return fail(ESMB200_EINVAL, "fp8 gemm epilogue must be 0 (qkv), 1 (residual) or 5 (gelu -> fp8)");
  }
  if (e != cudaSuccess) return fail_cuda(e, "gemm launch (fp8)");
  return ESMB200_OK;
}

inline int kblocks(int K) { return (K + 127) / 128; }  // 128-wide K blocks of the fp8 scales

// every GemmParams field an epilogue does not read stays zero
GemmParams gemm_params(int M, int N, int K, const float* bias) {
  GemmParams g;
  memset(&g, 0, sizeof g);
  g.M = M; g.N = N; g.K = K; g.bias = bias;
  return g;
}

// scratch layout of the attention kernels
struct AttnScratch {
  uint32_t* keybits;
  int* kvlen;
  float* row_max;
  float* row_sum;
  int words;
  size_t bytes;  // size of the whole layout
};

// the one definition of the layout: base 0 measures it (esmb200_attention_scratch_bytes), a device address carves it
AttnScratch attn_scratch_layout(uintptr_t base, int B, int T, int H) {
  AttnScratch s;
  s.words = (int)align_up((size_t)(T + 31) / 32, 4);
  const size_t keybits = align_up((size_t)B * s.words * 4, 256), kvlen = align_up((size_t)B * 4, 256);
  const size_t stats = align_up((size_t)B * H * T * 4, 256);
  s.keybits = reinterpret_cast<uint32_t*>(base);
  s.kvlen = reinterpret_cast<int*>(base + keybits);
  s.row_max = reinterpret_cast<float*>(base + keybits + kvlen);
  s.row_sum = reinterpret_cast<float*>(base + keybits + kvlen + stats);
  s.bytes = keybits + kvlen + 2 * stats;
  return s;
}

int run_key_bits(const uint8_t* pad_mask, const AttnScratch& s, int B, int T, cudaStream_t st) {
  const int wpb = 4;
  ProfScope ps(T_KEYBITS, st);
  key_bits_kernel<<<(B + wpb - 1) / wpb, wpb * 32, 0, st>>>(pad_mask, s.keybits, s.kvlen, B, T, s.words);
  CK(cudaGetLastError());
  return ESMB200_OK;
}

// contact-head accumulators of ONE layer (esmb200_contact_job resolved for layer i)
struct ContactLayer {
  const float* w;
  const uint8_t* keep;
  float* acc;
  float* row_part;
  float* col_part;
  int lo, S;
};

// attention_probs_kernel over the pp.B sequences: one launch (and one T_PROBS scope) per
// probs_cfg::seqs_per_launch(H) sequences, so a single launch whenever B*H <= 65535
int run_probs(const CUtensorMap& tq, ProbsParams pp, cudaStream_t st, const char* what) {
  const int per = probs_cfg::seqs_per_launch(pp.H);
  for (int b0 = 0; b0 < pp.B; b0 += per) {
    pp.b0 = b0;
    cudaError_t e;
    {
      ProfScope ps(T_PROBS, st);
      e = launch_attention_probs(tq, pp, pp.B - b0 < per ? pp.B - b0 : per, st);
    }
    if (e != cudaSuccess) return fail_cuda(e, what);
  }
  return ESMB200_OK;
}

int run_attention(const void* qkv, void* ctx, float* probs, long long probs_batch_stride, int attn_flags,
                  const AttnScratch& s, int B, int T, int H, cudaStream_t st, bool split = false,
                  const ContactLayer* contact = nullptr, int slots = 1) {
  const int E = H * 64 * slots;
  if (slots == 2 && split) return fail(ESMB200_EINVAL, "head_dim > 64: fp32x3 precision is not available");
  const uint64_t qcols = (uint64_t)(split ? 6 : 3) * E;  // fp32x3: [q k v]_hi | [q k v]_lo
  CUtensorMap tq;
  int rc = make_tmap_f16(&tq, qkv, (uint64_t)B * T, qcols, qcols, 128);
  if (rc) return rc;
  AttnParams ap;
  ap.B = B; ap.T = T; ap.H = H; ap.E = E;
  ap.lo_off = split ? 3 * E : 0;
  ap.slots = slots;
  ap.keybits = s.keybits; ap.kvlen = s.kvlen; ap.words = s.words;
  ap.ctx = static_cast<__half*>(ctx);
  ap.row_max = probs || contact ? s.row_max : nullptr;  // the contact pass reads them, with or without probs
  ap.row_sum = probs || contact ? s.row_sum : nullptr;
  cudaError_t e;
  {
    CUtensorMap tkv;
    rc = make_tmap_f16(&tkv, qkv, (uint64_t)B * T, qcols, qcols, attention_fwd_kv_box_rows(ap));
    if (rc) return rc;
    ProfScope ps(T_ATTN, st);
    e = launch_attention_fwd(tq, tkv, ap, num_sms(), st);
  }
  if (e != cudaSuccess) return fail_cuda(e, "attention launch");
  if (contact && !split) {
    // probabilities written once and folded into the contact accumulators in the same pass (attention_contact.cuh);
    // probs == nullptr: the same pass without the stores (esmb200_stack_contacts)
    if (B > 65535) return fail(ESMB200_EINVAL, "return_contacts: B must be <= 65535");
    ContactFuseParams cp;
    cp.B = B; cp.T = T; cp.H = H; cp.E = E; cp.slots = slots;
    cp.keybits = s.keybits; cp.kvlen = s.kvlen; cp.words = s.words;
    cp.row_max = s.row_max; cp.row_sum = s.row_sum; cp.probs = probs;
    cp.batch_stride = probs_batch_stride > 0 ? probs_batch_stride : (long long)H * T * T;
    cp.zero_pad_rows = attn_flags & 1;
    cp.w = contact->w; cp.keep = contact->keep; cp.acc = contact->acc;
    cp.row_part = contact->row_part; cp.col_part = contact->col_part; cp.lo = contact->lo; cp.S = contact->S;
    {
      ProfScope ps(T_PROBS, st);
      e = launch_attention_probs_contact(tq, cp, st);
    }
    if (e != cudaSuccess) return fail_cuda(e, "attention probs+contact launch");
    return ESMB200_OK;
  }
  if (probs) {
    ProbsParams pp;
    pp.B = B; pp.T = T; pp.H = H; pp.E = E;
    pp.keybits = s.keybits; pp.kvlen = s.kvlen; pp.words = s.words;
    pp.row_max = s.row_max; pp.row_sum = s.row_sum; pp.probs = probs;
    pp.batch_stride = probs_batch_stride > 0 ? probs_batch_stride : (long long)H * T * T;
    pp.zero_pad_rows = attn_flags & 1;
    pp.lo_off = split ? 3 * E : 0;
    pp.slots = slots;
    return run_probs(tq, pp, st, "attention probs launch");
  }
  return ESMB200_OK;
}

// contact_accumulate_kernel on one layer's maps (arguments validated by the caller: S = hi - lo <= 1024, B <= 65535)
int run_contact_accumulate(const float* attn, long long batch_stride, const float* w, const uint8_t* keep, float* acc,
                           float* row_sum, float* col_part, int B, int H, int T, int lo, int S, cudaStream_t st) {
  ProfScope ps(T_PROBS, st);
  const size_t smem = (size_t)8 * S * sizeof(float);
  dim3 grid((S + 15) / 16, B);  // 8 warps x 2 rows
  if (S <= 512)
    contact_accumulate_kernel<2, 16, 2><<<grid, 256, smem, st>>>(attn, batch_stride, w, keep, acc, row_sum, col_part, H, T,
                                                                  lo, S);
  else
    contact_accumulate_kernel<2, 32, 1><<<grid, 256, smem, st>>>(attn, batch_stride, w, keep, acc, row_sum, col_part, H, T,
                                                                  lo, S);
  CK(cudaGetLastError());
  return ESMB200_OK;
}

// MSA column attention (axial_attention.py:182-239) straight from the row-major qkv [B*R*C, 3E]: one "sequence" of R
// tokens per alignment column, read with strided TMA boxes (qkv viewed as [B*R, C*3E], AttnParams::cols), no
// regrouping copy.  s holds the key bits of the B*C column sequences.  split (fp32x3): qkv [B*R*C, 6E] (viewed as
// [B*R, C*6E], lo halves 3E to the right), ctx [B*R*C, 2E].  probs: optional fp32 [B*C, H, R, R], written from the
// same strided view with the row statistics of the forward kernel; ctx is the same with and without it.
int run_column_attention(const void* qkv, void* ctx, const AttnScratch& s, int B, int R, int C, int H,
                         cudaStream_t st, bool split = false, float* probs = nullptr) {
  const int E = H * 64;
  AttnParams ap;
  ap.B = B * C; ap.T = R; ap.H = H; ap.E = E;
  ap.lo_off = split ? 3 * E : 0;
  ap.keybits = s.keybits; ap.kvlen = s.kvlen; ap.words = s.words;
  ap.ctx = static_cast<__half*>(ctx);
  ap.row_max = probs ? s.row_max : nullptr;
  ap.row_sum = probs ? s.row_sum : nullptr;
  ap.cols = C;
  CUtensorMap tq, tkv;
  const uint64_t wide = (uint64_t)C * (split ? 6 : 3) * E;  // token r of column c at row r, x = c*3E (split: c*6E)
  int rc;
  if ((rc = make_tmap_f16(&tq, qkv, (uint64_t)B * R, wide, wide, 128))) return rc;
  if ((rc = make_tmap_f16(&tkv, qkv, (uint64_t)B * R, wide, wide, attention_fwd_kv_box_rows(ap)))) return rc;
  cudaError_t e;
  {
    ProfScope ps(T_ATTN, st);
    e = launch_attention_fwd(tq, tkv, ap, num_sms(), st);
  }
  if (e != cudaSuccess) return fail_cuda(e, "column attention launch");
  if (probs) {
    ProbsParams pp;
    pp.B = B * C; pp.T = R; pp.H = H; pp.E = E;
    pp.keybits = s.keybits; pp.kvlen = s.kvlen; pp.words = s.words;
    pp.row_max = s.row_max; pp.row_sum = s.row_sum; pp.probs = probs;
    pp.batch_stride = (long long)H * R * R;
    pp.zero_pad_rows = 0;
    pp.lo_off = ap.lo_off;
    pp.cols = C;
    return run_probs(tq, pp, st, "column attention probs launch");
  }
  return ESMB200_OK;
}

// LayerNorm -> fp16 GEMM operand [M, E], or with split the fp32x3 hi | lo halves [M, 2E]
int layernorm_f16(const float* x, const float* w, const float* b, void* out, int M, int E, float eps, bool split,
                  int tag, cudaStream_t st) {
  cudaError_t e;
  {
    ProfScope ps(tag, st);
    e = split ? launch_layernorm<2>(x, w, b, out, M, E, eps, st) : launch_layernorm<1>(x, w, b, out, M, E, eps, st);
  }
  if (e != cudaSuccess) return fail_cuda(e, split ? "layernorm_split" : "layernorm_f16");
  return ESMB200_OK;
}

// LayerNorm -> e4m3 GEMM operand [M, E] and its scales [ceil(E/128), M]
int layernorm_fp8(const float* x, const float* w, const float* b, void* out, float* scales, int M, int E, float eps,
                  int tag, cudaStream_t st) {
  cudaError_t e;
  {
    ProfScope ps(tag, st);
    e = launch_layernorm<3>(x, w, b, out, M, E, eps, st, scales);
  }
  if (e != cudaSuccess) return fail_cuda(e, "layernorm_fp8");
  return ESMB200_OK;
}

// fp32 [rows, K] -> e4m3 [rows, K] + scales per block_rows x 128 block (quantize_fp8_kernel)
int quantize_fp8(const float* src, uint8_t* dst, float* scales, int rows, int K, int block_rows, cudaStream_t st) {
  ProfScope ps(T_CONVERT, st);
  quantize_fp8_kernel<<<dim3(kblocks(K), (rows + block_rows - 1) / block_rows), 256, 0, st>>>(src, dst, scales, rows, K,
                                                                                               block_rows);
  CK(cudaGetLastError());
  return ESMB200_OK;
}

// fp32 [rows, K] -> fp16 [rows, K], or with split the fp32x3 hi | lo halves [rows, 2K]
int convert_f16(const float* src, void* dst, size_t rows, int K, bool split, cudaStream_t st) {
  const size_t n = rows * (size_t)K;
  size_t blocks = (n + 255) / 256;
  if (blocks > (size_t)num_sms() * 16) blocks = (size_t)num_sms() * 16;
  ProfScope ps(T_CONVERT, st);
  if (split)
    convert_f32_split_kernel<<<(unsigned)blocks, 256, 0, st>>>(src, static_cast<__half*>(dst), rows, K);
  else
    convert_f32_f16_kernel<<<(unsigned)blocks, 256, 0, st>>>(src, static_cast<__half*>(dst), n);
  CK(cudaGetLastError());
  return ESMB200_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// layer object
// ---------------------------------------------------------------------------------------------------------------
struct WeightMaps {
  CUtensorMap qkv, out, fc1, fc2;  // B operands, box {64, 128 rows}
};

struct esmb200_layer {
  int E, H, F;
  int d;          // head_dim (<= 128); every head occupies `slots` 64-wide slots of the attention-side tensors
  int slots;      // 1 (d <= 64) or 2 (64 < d <= 128, ESM-2 15B)
  int Ea;         // 64 * slots * H: width of q / k / v / ctx
  float q_scale;  // d^-1/2 (multihead_attention.py:100)
  int split;      // 1: fp32x3 precision — weights packed as fp16 hi | lo along K, activations likewise
  int fp8;        // 1: fp8 precision — QKV, fc1 and fc2 run the e4m3 GEMM from w8; out_proj stays fp16 (w_out)
  float eps;
  // borrowed fp32 parameters (owned by the caller, must outlive the layer)
  const float *ln1_w, *ln1_b, *ln2_w, *ln2_b, *out_b, *fc1_b, *fc2_b;
  // owned packed copies
  __half* w_qkv;  // [3*Ea, E]: row s*Ea + head_slot(h*d + j) <- W_s row h*d + j, zero rows elsewhere
  __half* w_out;  // [E, Ea]: column head_slot(h*d + j) <- out_proj.weight column h*d + j
  __half* w_fc1;  // [F,E]
  __half* w_fc2;  // [E,F]
  float* b_qkv;   // [3*Ea]
  // fp8 precision: one allocation holding the e4m3 matrices ([Wq;Wk;Wv] in head slots, fc1, fc2) and their 128 x 128
  // block scales (Fp8Layout); w_qkv, w_fc1 and w_fc2 stay NULL
  uint8_t* w8;
  uint8_t *q_qkv, *q_fc1, *q_fc2;
  float *s_qkv, *s_fc1, *s_fc2;
  WeightMaps tm;  // of w_qkv .. w_fc2; zero once offloaded
  // esmb200_layer_offload: the caller's pinned copy of w_qkv .. w_fc2 in the packed_layout() arrangement; the device
  // copies are freed and the layer runs only in esmb200_stack_forward_streamed
  const void* host;
};

namespace {
// one layer's packed matrices back to back, 1024-aligned: the layout of its host copy and of one ring slot
struct PackedLayout {
  size_t qkv, out, fc1, fc2;  // byte offsets
  size_t bytes;
};

PackedLayout packed_layout(int E, int H, int F, int split) {
  const size_t pf = split ? 2 : 1, Ea = (size_t)64 * head_slots(E, H) * H;
  PackedLayout p;
  p.qkv = 0;
  p.out = align_up(3 * Ea * E * 2 * pf, 1024);
  p.fc1 = p.out + align_up(Ea * E * 2 * pf, 1024);
  p.fc2 = p.fc1 + align_up((size_t)F * E * 2 * pf, 1024);
  p.bytes = p.fc2 + align_up((size_t)E * F * 2 * pf, 1024);
  return p;
}

// fp8 precision: the e4m3 matrices and their block scales [ceil(rows/128), ceil(K/128)] back to back, 1024-aligned
struct Fp8Layout {
  size_t qkv, fc1, fc2, s_qkv, s_fc1, s_fc2;  // byte offsets
  size_t bytes;
};

Fp8Layout fp8_layout(int E, int Ea, int F) {
  Fp8Layout l;
  size_t o = 0;
  auto take = [&](size_t n) {
    const size_t at = o;
    o += align_up(n, 1024);
    return at;
  };
  l.qkv = take((size_t)3 * Ea * E);
  l.fc1 = take((size_t)F * E);
  l.fc2 = take((size_t)E * F);
  l.s_qkv = take((size_t)kblocks(3 * Ea) * kblocks(E) * 4);
  l.s_fc1 = take((size_t)kblocks(F) * kblocks(E) * 4);
  l.s_fc2 = take((size_t)kblocks(E) * kblocks(F) * 4);
  l.bytes = o;
  return l;
}

// B-operand maps of a layer's fp8 matrices and its fp16 out_proj
int make_weight_maps_fp8(WeightMaps* m, const esmb200_layer* L) {
  int rc = make_tmap_2d(&m->qkv, L->q_qkv, 1, 3 * (uint64_t)L->Ea, L->E, L->E, gemm_fp8_cfg::BOX_ROWS);
  if (!rc) rc = make_tmap_f16(&m->out, L->w_out, L->E, L->Ea, L->Ea, gemm2_cfg::HALF_N);
  if (!rc) rc = make_tmap_2d(&m->fc1, L->q_fc1, 1, L->F, L->E, L->E, gemm_fp8_cfg::BOX_ROWS);
  if (!rc) rc = make_tmap_2d(&m->fc2, L->q_fc2, 1, L->E, L->F, L->F, gemm_fp8_cfg::BOX_ROWS);
  return rc;
}

// B-operand maps of a layer's packed matrices (fc1 == nullptr: attention-only layer)
int make_weight_maps(WeightMaps* m, const __half* qkv, const __half* out, const __half* fc1, const __half* fc2, int E,
                     int Ea, int F, int split) {
  const uint64_t pf = split ? 2 : 1;
  const uint32_t wbox = gemm2_cfg::HALF_N;
  int rc = make_tmap_f16(&m->qkv, qkv, 3 * (uint64_t)Ea, pf * E, pf * E, wbox);
  if (!rc) rc = make_tmap_f16(&m->out, out, E, pf * Ea, pf * Ea, wbox);
  if (!rc && fc1) rc = make_tmap_f16(&m->fc1, fc1, F, pf * E, pf * E, wbox);
  if (!rc && fc1) rc = make_tmap_f16(&m->fc2, fc2, E, pf * F, pf * F, wbox);
  return rc;
}

struct Workspace {
  __half* xn;    // fp8 precision: e4m3 [M,E], followed by its scales xn_s [ceil(E/128), M]
  __half* qkv;
  __half* ctx;
  __half* h;     // aliases qkv + ctx; fp8 precision: e4m3 [M,F], followed by its scales h_s [F/128, M]
  float* xn_s;
  float* h_s;
  AttnScratch as;
  size_t bytes;  // size of the whole layout, including 1024 bytes to align the caller's pointer
};

// the one definition of the layer workspace: nullptr measures it (esmb200_workspace_bytes), a device pointer carves it.
// precision 2 (fp8): xn and h are e4m3 with their scale arrays behind them; q, k, v and ctx stay fp16.
Workspace workspace_layout(void* workspace, int E, int H, int F, int B, int T, int precision) {
  const bool fp8 = precision == 2;
  const size_t M = (size_t)B * T, Ea = (size_t)64 * head_slots(E, H) * H, pf = precision && !fp8 ? 2 : 1;
  const uintptr_t base = workspace ? align_up(reinterpret_cast<uintptr_t>(workspace), 1024) : 0;
  const size_t xn_q = fp8 ? align_up(M * E, 1024) : 0, h_q = fp8 ? align_up(M * F, 1024) : 0;
  const size_t xn = fp8 ? xn_q + align_up((size_t)kblocks(E) * M * 4, 1024)
                        : align_up(M * E * 2 * pf, 1024);  // fp16 [M,E] (hi | lo)
  const size_t qkv = align_up(M * 3 * Ea * 2 * pf, 1024), ctx = align_up(M * Ea * 2 * pf, 1024);
  const size_t h = fp8 ? h_q + align_up((size_t)kblocks(F) * M * 4, 1024) : align_up(M * F * 2 * pf, 1024);
  const size_t scratch = xn + (qkv + ctx > h ? qkv + ctx : h);
  Workspace ws;
  ws.xn = reinterpret_cast<__half*>(base);
  ws.qkv = ws.h = reinterpret_cast<__half*>(base + xn);
  ws.ctx = reinterpret_cast<__half*>(base + xn + qkv);
  ws.xn_s = fp8 ? reinterpret_cast<float*>(base + xn_q) : nullptr;
  ws.h_s = fp8 ? reinterpret_cast<float*>(base + xn + h_q) : nullptr;
  ws.as = attn_scratch_layout(base + scratch, B, T, H);
  ws.bytes = scratch + ws.as.bytes + 1024;
  return ws;
}

struct ActMaps {
  CUtensorMap xn, ctx, h;       // A operands (fp16, box {64,128})
  CUtensorMap qkv_o, h_o, x_o;  // GEMM outputs: qkv and h (fp16), the fp32 residual stream x
};

// The QKV projection of a layer of E = H d: N = 3 Ea columns in head slots (Ea = 64 slots H), K = E, the q columns scaled
// by q_scale, q and k rotated per 64-wide slot by a [T, 32 slots] table when rope_cos is given, the fp32x3 lo halves
// 3 Ea columns to the right.  attention_block and esmb200_gemm_qkv_heads launch the projection with these parameters.
GemmParams qkv_params(int M, int E, int Ea, int slots, const float* bias, const float* rope_cos, const float* rope_sin,
                      int T, float q_scale) {
  GemmParams g = gemm_params(M, 3 * Ea, E, bias);
  g.rope_cos = rope_cos; g.rope_sin = rope_sin; g.rope_ld = 32 * slots; g.T = T; g.E = Ea; g.q_scale = q_scale;
  g.lo_col_off = 3 * Ea;
  return g;
}

// x += out_proj(attend()) after LN1 -> fp16 and the q,k,v projection (+ bias, q scale, RoPE when rope_cos is given):
// the self-attention half of an ESM-2 layer (multihead_attention.py:258-261,354-355,395; modules.py:124-134) and each
// axial attention sub-layer of the MSA stack.  `attend` reads ws.qkv and writes ws.ctx.  The weights are read through
// `wm`: the layer's own maps (L->tm), or those of the ring slot its packed matrices were streamed into.
template <class Attend>
int attention_block(const esmb200_layer* L, const WeightMaps& wm, float* x, int M, int T, const float* rope_cos,
                    const float* rope_sin, float q_scale, const Workspace& ws, const ActMaps& am, cudaStream_t st,
                    Attend attend) {
  const bool split = L->split != 0;
  int rc = L->fp8 ? layernorm_fp8(x, L->ln1_w, L->ln1_b, ws.xn, ws.xn_s, M, L->E, L->eps, T_LN1, st)
                  : layernorm_f16(x, L->ln1_w, L->ln1_b, ws.xn, M, L->E, L->eps, split, T_LN1, st);
  if (rc) return rc;
  const GemmParams g = qkv_params(M, L->E, L->Ea, L->slots, L->b_qkv, rope_cos, rope_sin, T, q_scale);
  rc = L->fp8 ? launch_gemm_fp8(EPI_QKV_ROPE, am.xn, wm.qkv, am.qkv_o, {g, ws.xn_s, L->s_qkv, nullptr}, st, T_QKV)
              : launch_gemm(EPI_QKV_ROPE, am.xn, wm.qkv, am.qkv_o, g, st, T_QKV, split);
  if (rc) return rc;
  if ((rc = attend())) return rc;
  return launch_gemm(EPI_BIAS_RESIDUAL, am.ctx, wm.out, am.x_o, gemm_params(M, L->E, L->Ea, L->out_b), st, T_OUT,
                     split);
}

// x += fc2(GELU(fc1(LN2(x)))) (modules.py:137-140, 413-418)
int ffn_block(const esmb200_layer* L, const WeightMaps& wm, float* x, int M, const Workspace& ws, const ActMaps& am,
              cudaStream_t st) {
  const bool split = L->split != 0;
  if (L->fp8) {
    int rc = layernorm_fp8(x, L->ln2_w, L->ln2_b, ws.xn, ws.xn_s, M, L->E, L->eps, T_LN2, st);
    if (!rc)
      rc = launch_gemm_fp8(EPI_GELU_FP8, am.xn, wm.fc1, am.h_o, {gemm_params(M, L->F, L->E, L->fc1_b), ws.xn_s,
                                                                  L->s_fc1, ws.h_s}, st, T_FC1);
    if (!rc)
      rc = launch_gemm_fp8(EPI_BIAS_RESIDUAL, am.h, wm.fc2, am.x_o, {gemm_params(M, L->E, L->F, L->fc2_b), ws.h_s,
                                                                      L->s_fc2, nullptr}, st, T_FC2);
    return rc;
  }
  int rc = layernorm_f16(x, L->ln2_w, L->ln2_b, ws.xn, M, L->E, L->eps, split, T_LN2, st);
  if (rc) return rc;
  GemmParams g = gemm_params(M, L->F, L->E, L->fc1_b);
  g.lo_col_off = L->F;
  if ((rc = launch_gemm(EPI_BIAS_GELU, am.xn, wm.fc1, am.h_o, g, st, T_FC1, split))) return rc;
  return launch_gemm(EPI_BIAS_RESIDUAL, am.h, wm.fc2, am.x_o, gemm_params(M, L->E, L->F, L->fc2_b), st, T_FC2,
                     split);
}

// precision 0 fp16, 1 fp32x3, 2 fp8 (xn and h e4m3)
int make_act_maps(ActMaps* am, const Workspace& ws, float* x, int E, int H, int F, int M, int precision = 0) {
  // fp32x3: activations are [rows, 2 * width]
  const uint64_t Ea = (uint64_t)64 * head_slots(E, H) * H, pf = precision == 1 ? 2 : 1;
  const int es = precision == 2 ? 1 : 2;  // element bytes of xn and h
  // xn and h feed the fp8 GEMM in precision 2: its producer expects boxes of gemm_fp8_cfg::BOX_ROWS rows
  const uint32_t box = precision == 2 ? gemm_fp8_cfg::BOX_ROWS : gemm2_cfg::BOX_M;
  int rc = make_tmap_2d(&am->xn, ws.xn, es, M, pf * E, pf * E, box);
  if (!rc) rc = make_tmap_f16(&am->ctx, ws.ctx, M, pf * Ea, pf * Ea, gemm2_cfg::BOX_M);
  if (!rc) rc = make_tmap_2d(&am->h, ws.h, es, M, pf * F, pf * F, box);
  if (!rc) rc = make_gemm_out_map(&am->qkv_o, ws.qkv, 2, M, pf * 3 * Ea);
  if (!rc) rc = make_gemm_out_map(&am->h_o, ws.h, es, M, pf * F);
  if (!rc) rc = make_gemm_out_map(&am->x_o, x, 4, M, E);
  return rc;
}

// The standalone GEMMs: out = epilogue(a . w^T + bias) with a [M, K] and w [N, K] fp16, or with split their fp32x3
// hi | lo halves [M, 2K] and [N, 2K] and an fp16 output as hi | lo [M, 2N].  The arguments are validated by the caller.
int run_gemm(int epi, const void* a, const void* w, const float* bias, void* out, int M, int N, int K,
             const float* rope_cos, const float* rope_sin, int T, int E, float q_scale, bool split, void* stream) {
  const bool f16_out = (epi == EPI_QKV_ROPE || epi == EPI_BIAS_GELU);
  const uint64_t pf = split ? 2 : 1;
  CUtensorMap ta, tb, to;
  int rc = make_tmap_f16(&ta, a, M, pf * K, pf * K, gemm2_cfg::BOX_M);
  if (!rc) rc = make_tmap_f16(&tb, w, N, pf * K, pf * K, gemm2_cfg::HALF_N);
  if (!rc) rc = f16_out ? make_gemm_out_map(&to, out, 2, M, pf * N) : make_gemm_out_map(&to, out, 4, M, N);
  if (rc) return rc;
  GemmParams g = gemm_params(M, N, K, bias);
  g.rope_cos = rope_cos; g.rope_sin = rope_sin; g.T = T; g.E = E; g.q_scale = q_scale;
  g.lo_col_off = N;
  return launch_gemm(epi, ta, tb, to, g, static_cast<cudaStream_t>(stream), T_GEMM_OTHER, split);
}

// esmb200_gemm_f16 and esmb200_gemm_split
int gemm_epilogue_entry(int epi, const void* a, const void* w, const float* bias, void* out, int M, int N, int K,
                        const float* rope_cos, const float* rope_sin, int T, int E, bool split, void* stream) {
  if (!a || !w || !bias || !out) return fail(ESMB200_EINVAL, "null argument");
  const bool f16_out = (epi == EPI_QKV_ROPE || epi == EPI_BIAS_GELU);
  if (M <= 0 || N <= 0 || K <= 0 || K % (split ? 64 : 8) != 0 || N % (f16_out ? 64 : 32) != 0)
    return fail(ESMB200_EINVAL, std::string(split ? "split gemm needs K % 64 == 0" : "gemm needs K % 8 == 0") +
                                    " and N % 64 == 0 (fp16 output) / N % 32 == 0 (fp32 output)");
  if (split && (epi < 0 || epi > EPI_BIAS_GELU_F32)) return fail(ESMB200_EINVAL, "unknown GEMM epilogue");
  int rc = check_device();
  if (rc) return rc;
  if (epi == EPI_QKV_ROPE && (!rope_cos || !rope_sin || T <= 0 || E <= 0 || E % 64 != 0 || N != 3 * E))
    return fail(ESMB200_EINVAL, "qkv epilogue needs rope tables, T and N == 3E");
  return run_gemm(epi, a, w, bias, out, M, N, K, rope_cos, rope_sin, T, E, 0.125f, split, stream);
}

// esmb200_attention (head_dim <= 64), esmb200_attention128 (slots = 2) and esmb200_attention_split (fp32x3)
int attention_entry(const void* qkv, const uint8_t* pad_mask, void* ctx, float* attn_probs, int B, int T, int H,
                    void* scratch, void* stream, bool split, int slots) {
  if (!qkv || !ctx || !scratch) return fail(ESMB200_EINVAL, "null argument");
  if (B <= 0 || T <= 0 || H <= 0 || H > 64) return fail(ESMB200_EINVAL, "bad shape");
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const AttnScratch s = attn_scratch_layout(reinterpret_cast<uintptr_t>(scratch), B, T, H);
  rc = run_key_bits(pad_mask, s, B, T, st);
  if (rc) return rc;
  return run_attention(qkv, ctx, attn_probs, 0, 0, s, B, T, H, st, split, nullptr, slots);
}

// MSA stack workspace: the layer workspace of the B*C column sequences of R tokens, then the tied row-attention scratch
struct AxialWorkspace {
  Workspace ws;
  uint8_t* tied;
  size_t tied_bytes;
  size_t bytes;
};

// scratch of the tied row attention: fp32 logits [H,B,C,C], then P [H*B*C, Cp] fp16 (split: hi | lo, [H*B*C, 2*Cp])
size_t tied_scratch_bytes(int B, int C, int H, int split) {
  const size_t Cp = align_up((size_t)C, 64), pf = split ? 2 : 1;
  return align_up((size_t)H * B * C * C * 4, 1024) + align_up((size_t)H * B * C * Cp * 2 * pf, 1024) + 2048;
}

// the one definition of the MSA stack workspace: nullptr measures it (esmb200_axial_workspace_bytes and its _split
// variant), a device pointer carves it
AxialWorkspace axial_workspace_layout(void* workspace, int E, int F, int B, int R, int C, int split) {
  AxialWorkspace a;
  a.ws = workspace_layout(workspace, E, E / 64, F, B * C, R, split);
  a.tied = reinterpret_cast<uint8_t*>(a.ws.xn) + a.ws.bytes;
  a.tied_bytes = tied_scratch_bytes(B, C, E / 64, split);
  a.bytes = a.ws.bytes + a.tied_bytes + 1024;
  return a;
}

// esmb200_stack_forward_streamed: two device slots that the offloaded layers' packed matrices are copied into on `copy`
// (layer i into slot i % 2), with the events that order the copies against the layers reading the slots
struct WeightRing {
  cudaStream_t st = nullptr, copy = nullptr;
  uint8_t* slot[2] = {};
  size_t bytes = 0;               // one layer's packed matrices
  WeightMaps maps[2];
  cudaEvent_t copied[2] = {}, freed[2] = {}, mark = nullptr;
  // the caller's stream waits for the last copy: an error can leave the layer loop before the wait for a copy that
  // is still writing the ring, which the caller may free or reuse in stream order once the call returns
  ~WeightRing() {
    if (mark && cudaEventRecord(mark, copy) == cudaSuccess) cudaStreamWaitEvent(st, mark, 0);
    for (cudaEvent_t e : {copied[0], copied[1], freed[0], freed[1], mark})
      if (e) cudaEventDestroy(e);
  }
  int init(uint8_t* ring, size_t layer_bytes, cudaStream_t stream, cudaStream_t copy_stream) {
    st = stream; copy = copy_stream; bytes = layer_bytes;
    slot[0] = ring; slot[1] = ring + layer_bytes;
    for (cudaEvent_t* e : {&copied[0], &copied[1], &freed[0], &freed[1], &mark})
      CK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    // a previous call on `stream` may still be reading a slot of the same ring
    CK(cudaEventRecord(mark, st));
    CK(cudaStreamWaitEvent(copy, mark, 0));
    return ESMB200_OK;
  }
  // layer i's packed matrices -> slot i % 2, once layer i - 2 (the last reader of that slot) has run
  int fetch(const esmb200_layer* L, int i) {
    const int s = i & 1;
    if (i >= 2) CK(cudaStreamWaitEvent(copy, freed[s], 0));
    CK(cudaMemcpyAsync(slot[s], L->host, bytes, cudaMemcpyHostToDevice, copy));
    CK(cudaEventRecord(copied[s], copy));
    return ESMB200_OK;
  }
};
}  // namespace

extern "C" {

int esmb200_abi_version(void) { return ESMB200_ABI_VERSION; }

const char* esmb200_last_error(void) { return g_last_error.c_str(); }

int esmb200_convert_f16(const float* src, void* dst, size_t n, void* stream) {
  if (n == 0) return ESMB200_OK;
  return convert_f16(src, dst, n, 1, false, static_cast<cudaStream_t>(stream));
}

int esmb200_layer_destroy(esmb200_layer* L) {
  if (!L) return ESMB200_OK;
  cudaFree(L->w_qkv);
  cudaFree(L->w_out);
  cudaFree(L->w_fc1);
  cudaFree(L->w_fc2);
  cudaFree(L->b_qkv);
  cudaFree(L->w8);
  delete L;
  return ESMB200_OK;
}

int esmb200_layer_create(const esmb200_layer_weights* w, void* stream, esmb200_layer** out) {
  if (!w || !out) return fail(ESMB200_EINVAL, "null argument");
  int rc = check_device();
  if (rc) return rc;
  const int E = w->embed_dim, H = w->num_heads, F = w->ffn_dim;
  if (E <= 0 || H <= 0 || E % H != 0) return fail(ESMB200_EINVAL, "embed_dim must be a positive multiple of num_heads");
  const int d = w->head_dim > 0 ? w->head_dim : E / H;
  if (d * H != E || d > 128 || d % 2 != 0)
    return fail(ESMB200_EINVAL, "esmb200 supports even head_dim <= 128 (every ESM-2 model, MSA Transformer)");
  if (E % 16 != 0) return fail(ESMB200_EINVAL, "embed_dim must be a multiple of 16");
  const bool has_ffn = w->fc1_weight != nullptr;  // NULL fc1_weight: attention-only layer (MSA row-attention sub-layer)
  if (has_ffn && (F <= 0 || F % 64 != 0)) return fail(ESMB200_EINVAL, "ffn_dim must be a positive multiple of 64");
  if (w->precision < 0 || w->precision > 2)
    return fail(ESMB200_EINVAL,
                "precision must be 0 (fp16 operands), 1 (fp32x3: fp16 hi|lo operands) or 2 (fp8: e4m3 QKV/fc1/fc2)");
  if (w->precision == 2 && (!has_ffn || F % 128 != 0))
    return fail(ESMB200_EINVAL, "fp8 precision needs a feed-forward layer with ffn_dim % 128 == 0 (ESM-2, ESM-1b/1v)");
  const int split = w->precision == 1;
  const int fp8 = w->precision == 2;
  const int slots = head_slots(E, H);
  if (split && slots == 2) return fail(ESMB200_EINVAL, "fp32x3 precision is not available for head_dim > 64");
  if (split && E % 64 != 0)
    return fail(ESMB200_EINVAL, "fp32x3 precision needs embed_dim % 64 == 0 (all ESM-2 models except 35M)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  esmb200_layer* L = new esmb200_layer();
  memset(static_cast<void*>(L), 0, sizeof(*L));
  const int Ea = 64 * slots * H;
  L->E = E; L->H = H; L->F = has_ffn ? F : 0; L->d = d; L->slots = slots; L->Ea = Ea; L->eps = w->ln_eps;
  // the reference's head_dim ** -0.5 is a Python double, rounded to fp32 by `q *= scaling`; 1.0f / sqrtf(d) in fp32
  // is one ulp off at d = 6, 18, 24 (esm2_t12_35M), 28, 34, 58, 68, 72, ... (DESIGN.md section 4)
  L->q_scale = (float)pow((double)d, -0.5);
  L->ln1_w = w->ln1_weight; L->ln1_b = w->ln1_bias; L->ln2_w = w->ln2_weight; L->ln2_b = w->ln2_bias;
  L->out_b = w->out_bias; L->fc1_b = w->fc1_bias; L->fc2_b = w->fc2_bias;
  L->split = split;
  L->fp8 = fp8;
  const size_t pf = split ? 2 : 1;  // fp32x3: every K extent doubles (hi | lo)
  const size_t EaE = (size_t)Ea * E, EF = (size_t)E * F;
  cudaError_t e;
#define ALLOC(ptr, bytes)                                              \
  if ((e = cudaMalloc(reinterpret_cast<void**>(&(ptr)), (bytes))) != cudaSuccess) { \
    esmb200_layer_destroy(L);                                          \
    return fail_cuda(e, "cudaMalloc(packed weights)");                 \
  }
  const Fp8Layout fl = fp8_layout(E, Ea, F);
  if (fp8) {
    ALLOC(L->w8, fl.bytes);
    L->q_qkv = L->w8 + fl.qkv; L->q_fc1 = L->w8 + fl.fc1; L->q_fc2 = L->w8 + fl.fc2;
    L->s_qkv = reinterpret_cast<float*>(L->w8 + fl.s_qkv);
    L->s_fc1 = reinterpret_cast<float*>(L->w8 + fl.s_fc1);
    L->s_fc2 = reinterpret_cast<float*>(L->w8 + fl.s_fc2);
  } else {
    ALLOC(L->w_qkv, 3 * EaE * 2 * pf);
  }
  ALLOC(L->w_out, EaE * 2 * pf);
  if (has_ffn && !fp8) {
    ALLOC(L->w_fc1, EF * 2 * pf);
    ALLOC(L->w_fc2, EF * 2 * pf);
  }
  ALLOC(L->b_qkv, (size_t)3 * Ea * 4);
#undef ALLOC
  // every head goes into its zero-padded 64-wide slot(s) (elementwise.cuh head_slot; for head_dim 64 the identity)
  e = fp8 ? cudaSuccess : cudaMemsetAsync(L->w_qkv, 0, 3 * EaE * 2 * pf, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(L->w_out, 0, EaE * 2 * pf, st);
  if (e == cudaSuccess) e = cudaMemsetAsync(L->b_qkv, 0, (size_t)3 * Ea * 4, st);
  if (e != cudaSuccess) rc = fail_cuda(e, "memset(packed weights)");
  const float* ws3[3] = {w->q_weight, w->k_weight, w->v_weight};
  const float* bs3[3] = {w->q_bias, w->k_bias, w->v_bias};
  const unsigned blocks = (unsigned)(((size_t)E * E + 255) / 256);
  if (fp8 && !rc) {
    // [Wq;Wk;Wv] into their head slots as fp32, then 128 x 128 block quantisation; fc1 and fc2 straight from the caller
    float* staged = nullptr;
    e = cudaMallocAsync(reinterpret_cast<void**>(&staged), 3 * EaE * 4, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(staged, 0, 3 * EaE * 4, st);
    for (int s3 = 0; s3 < 3 && e == cudaSuccess; ++s3) {
      ProfScope ps(T_CONVERT, st);
      pack_head_rows_f32_kernel<<<blocks, 256, 0, st>>>(ws3[s3], bs3[s3], staged + (size_t)s3 * EaE,
                                                        L->b_qkv + s3 * Ea, E, d);
      e = cudaGetLastError();
    }
    if (e != cudaSuccess) rc = fail_cuda(e, "pack_head_rows (fp8)");
    if (!rc) rc = quantize_fp8(staged, L->q_qkv, L->s_qkv, 3 * Ea, E, 128, st);
    if (staged) cudaFreeAsync(staged, st);
    if (!rc) rc = quantize_fp8(w->fc1_weight, L->q_fc1, L->s_fc1, F, E, 128, st);
    if (!rc) rc = quantize_fp8(w->fc2_weight, L->q_fc2, L->s_fc2, E, F, 128, st);
  }
  for (int s3 = 0; s3 < 3 && !rc && !fp8; ++s3) {
    ProfScope ps(T_CONVERT, st);
    pack_head_rows_kernel<<<blocks, 256, 0, st>>>(ws3[s3], bs3[s3], L->w_qkv + (size_t)s3 * EaE * pf, L->b_qkv + s3 * Ea,
                                                  E, d, split);
    if ((e = cudaGetLastError()) != cudaSuccess) rc = fail_cuda(e, "pack_head_rows");
  }
  if (!rc) {
    ProfScope ps(T_CONVERT, st);
    pack_head_cols_kernel<<<blocks, 256, 0, st>>>(w->out_weight, L->w_out, E, Ea, d, split);
    if ((e = cudaGetLastError()) != cudaSuccess) rc = fail_cuda(e, "pack_head_cols");
  }
  if (!rc && has_ffn && !fp8) rc = convert_f16(w->fc1_weight, L->w_fc1, F, E, split, st);
  if (!rc && has_ffn && !fp8) rc = convert_f16(w->fc2_weight, L->w_fc2, E, F, split, st);
  if (!rc) rc = fp8 ? make_weight_maps_fp8(&L->tm, L)
                    : make_weight_maps(&L->tm, L->w_qkv, L->w_out, L->w_fc1, L->w_fc2, E, Ea, L->F, split);
  if (rc) {
    esmb200_layer_destroy(L);
    return rc;
  }
  *out = L;
  return ESMB200_OK;
}

size_t esmb200_attention_scratch_bytes(int32_t B, int32_t T) {
  // H is bounded by E/64; the stats arrays are sized by the caller-visible worst case through workspace_bytes,
  // this standalone entry sizes them for H <= 64.
  return attn_scratch_layout(0, B, T, 64).bytes;
}

size_t esmb200_workspace_bytes(int32_t E, int32_t H, int32_t F, int32_t B, int32_t T, int32_t precision) {
  return workspace_layout(nullptr, E, H, F, B, T, precision).bytes;
}

size_t esmb200_layer_packed_bytes(int32_t E, int32_t H, int32_t F, int32_t precision) {
  if (E <= 0 || H <= 0 || F <= 0 || E % H != 0 || E / H > 128 || (precision != 0 && precision != 1)) return 0;
  return packed_layout(E, H, F, precision).bytes;
}

int esmb200_layer_offload(esmb200_layer* L, void* host_dst, size_t bytes, void* stream) {
  if (!L || !host_dst) return fail(ESMB200_EINVAL, "null argument");
  if (L->host) return fail(ESMB200_EINVAL, "layer is already offloaded");
  if (L->F <= 0) return fail(ESMB200_EINVAL, "attention-only layers cannot be offloaded");
  if (L->fp8) return fail(ESMB200_EINVAL, "fp8 layers cannot be offloaded: streamed layers run fp16 or fp32x3");
  const PackedLayout p = packed_layout(L->E, L->H, L->F, L->split);
  if (bytes < p.bytes) return fail(ESMB200_EINVAL, "host buffer smaller than esmb200_layer_packed_bytes");
  int rc = check_device();
  if (rc) return rc;
  cudaPointerAttributes pa;
  if (cudaPointerGetAttributes(&pa, host_dst) != cudaSuccess || pa.type != cudaMemoryTypeHost) {
    cudaGetLastError();
    return fail(ESMB200_EINVAL, "host_dst must be pinned host memory (cudaHostAlloc / cudaHostRegister)");
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* h = static_cast<uint8_t*>(host_dst);
  const size_t pf = L->split ? 2 : 1, EaE = (size_t)L->Ea * L->E, EF = (size_t)L->E * L->F;
  CK(cudaMemcpyAsync(h + p.qkv, L->w_qkv, 3 * EaE * 2 * pf, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h + p.out, L->w_out, EaE * 2 * pf, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h + p.fc1, L->w_fc1, EF * 2 * pf, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(h + p.fc2, L->w_fc2, EF * 2 * pf, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));  // the copies read what is freed below
  for (__half** w : {&L->w_qkv, &L->w_out, &L->w_fc1, &L->w_fc2}) {
    cudaFree(*w);
    *w = nullptr;
  }
  memset(&L->tm, 0, sizeof L->tm);
  L->host = host_dst;
  return ESMB200_OK;
}

// esmb200_stack_contacts: the partial buffers of a contact job and the fp32x3 probability scratch, in bytes
struct ContactSizes {
  size_t row_part, col_part, scratch;
};

static ContactSizes contact_sizes(int n_layers, int H, int B, int T, int S, int precision) {
  const size_t lbh = (size_t)n_layers * B * H;
  ContactSizes c;
  if (precision == 1) {  // fp32x3: contact_accumulate_kernel's row sums and 16-row column stripes, one layer's maps
    c.row_part = lbh * S * 4;
    c.col_part = lbh * ((S + 15) / 16) * S * 4;
    c.scratch = (size_t)B * H * T * T * 4;
  } else {  // the fused pass: one partial per 32-key / 32-query quarter of each 128-wide tile
    c.row_part = c.col_part = lbh * 4 * ((T + 127) / 128) * S * 4;
    c.scratch = 0;
  }
  return c;
}

// the layer loop of esmb200_stack_forward (ring == nullptr: every layer's weights resident), of
// esmb200_stack_forward_streamed (every layer offloaded, its packed matrices copied into `ring` ahead of use) and, with
// contacts_only, of esmb200_stack_contacts (attn_out == nullptr; fp32x3 maps go through `scratch` one layer at a time)
static int stack_forward_impl(esmb200_layer* const* layers, int32_t n_layers, float* x, const uint8_t* pad_mask,
                              int32_t B, int32_t T, const float* rope_cos, const float* rope_sin,
                              float* const* repr_out, float* const* attn_out, int64_t attn_batch_stride,
                              int32_t attn_flags, const esmb200_contact_job* contact, void* workspace,
                              size_t workspace_bytes, void* ring, size_t ring_bytes, void* copy_stream, void* stream,
                              bool contacts_only = false, void* scratch = nullptr, size_t scratch_bytes = 0) {
  if (!layers || n_layers <= 0 || !x || !workspace) return fail(ESMB200_EINVAL, "null argument");
  for (int i = 0; i < n_layers; ++i)
    if (!layers[i]) return fail(ESMB200_EINVAL, "null layer");
  if ((rope_cos == nullptr) != (rope_sin == nullptr))  // both NULL: no rotary embedding (ESM-1b / ESM-1v)
    return fail(ESMB200_EINVAL, "rope_cos and rope_sin must both be given or both be NULL");
  if (contacts_only && !contact) return fail(ESMB200_EINVAL, "null contact job");
  if (contact) {
    if (!contacts_only && !attn_out) return fail(ESMB200_EINVAL, "a contact job needs attn_out for every layer");
    for (int i = 0; i < n_layers && !contacts_only; ++i)
      if (!attn_out[i]) return fail(ESMB200_EINVAL, "a contact job needs attn_out for every layer");
    if (!contact->weights || !contact->acc || !contact->row_part || !contact->col_part || contact->lo < 0 ||
        contact->hi > T || contact->hi <= contact->lo)
      return fail(ESMB200_EINVAL, "bad contact job");
  }
  if (B <= 0 || T <= 0) return fail(ESMB200_EINVAL, "empty batch");
  if ((long long)B * T > 0x7fffffffLL / 8) return fail(ESMB200_EINVAL, "B*T too large for one call; split the batch");
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int E = layers[0]->E, F = layers[0]->F, H = layers[0]->H;
  if (F <= 0) return fail(ESMB200_EINVAL, "attention-only layers belong to esmb200_axial_stack_forward");
  for (int i = 1; i < n_layers; ++i)
    if (layers[i]->E != E || layers[i]->F != F || layers[i]->H != H || layers[i]->split != layers[0]->split ||
        layers[i]->fp8 != layers[0]->fp8)
      return fail(ESMB200_EINVAL, "layers of one stack must share E, H, F and precision");
  const bool streamed = ring != nullptr;
  for (int i = 0; i < n_layers; ++i)
    if ((layers[i]->host != nullptr) != streamed)
      return fail(ESMB200_EINVAL, "layer " + std::to_string(i) +
                                      (streamed ? " is not offloaded: esmb200_stack_forward_streamed runs layers "
                                                  "whose weights esmb200_layer_offload moved to host memory"
                                                : " is offloaded to host memory (esmb200_layer_offload): run it with "
                                                  "esmb200_stack_forward_streamed"));
  const int split = layers[0]->split;
  const int precision = layers[0]->fp8 ? 2 : split;
  const Workspace ws = workspace_layout(workspace, E, H, F, B, T, precision);
  if (workspace_bytes < ws.bytes) return fail(ESMB200_EWORKSPACE, "workspace too small");
  const int S = contact ? contact->hi - contact->lo : 0;
  if (contacts_only) {  // refused before anything is launched
    if (B > 65535) return fail(ESMB200_EINVAL, "return_contacts: B must be <= 65535");
    if (split) {
      if (S > kContactMaxS) return fail(ESMB200_EINVAL, kContactMaxSMsg);
      if (!scratch || scratch_bytes < contact_sizes(n_layers, H, B, T, S, precision).scratch)
        return fail(ESMB200_EWORKSPACE, "probability scratch smaller than esmb200_stack_contacts_bytes");
      if (reinterpret_cast<uintptr_t>(scratch) % 16 != 0)
        return fail(ESMB200_EINVAL, "probability scratch must be 16-byte aligned");
    }
  }
  ActMaps am;
  rc = make_act_maps(&am, ws, x, E, H, F, B * T, precision);
  if (rc) return rc;
  WeightRing wr;
  if (streamed) {
    const PackedLayout p = packed_layout(E, H, F, split);
    if (ring_bytes < 2 * p.bytes) return fail(ESMB200_EINVAL, "ring smaller than 2 * esmb200_layer_packed_bytes");
    uint8_t* base = static_cast<uint8_t*>(ring);
    const int Ea = layers[0]->Ea;
    for (int s = 0; s < 2 && !rc; ++s) {
      uint8_t* b = base + s * p.bytes;
      rc = make_weight_maps(&wr.maps[s], reinterpret_cast<__half*>(b + p.qkv), reinterpret_cast<__half*>(b + p.out),
                            reinterpret_cast<__half*>(b + p.fc1), reinterpret_cast<__half*>(b + p.fc2), E, Ea, F, split);
    }
    if (rc) return rc;
    if ((rc = wr.init(base, p.bytes, st, static_cast<cudaStream_t>(copy_stream)))) return rc;
    for (int i = 0; i < 2 && i < n_layers && !rc; ++i) rc = wr.fetch(layers[i], i);
    if (rc) return rc;
  }
  rc = run_key_bits(pad_mask, ws.as, B, T, st);
  if (rc) return rc;
  const int nt128 = (T + 127) / 128;
  for (int i = 0; i < n_layers; ++i) {
    esmb200_layer* L = layers[i];
    const WeightMaps* wm = &L->tm;
    if (streamed) {
      CK(cudaStreamWaitEvent(st, wr.copied[i & 1], 0));
      wm = &wr.maps[i & 1];
    }
    ContactLayer cl;
    if (contact) {
      const size_t part = (size_t)B * H * nt128 * S;
      cl.w = contact->weights + (size_t)i * H; cl.keep = contact->keep; cl.acc = contact->acc;
      cl.row_part = contact->row_part + (size_t)i * 4 * part; cl.col_part = contact->col_part + (size_t)i * 4 * part;
      cl.lo = contact->lo; cl.S = S;
    }
    float* probs = attn_out ? attn_out[i] : nullptr;
    if (contacts_only && split) {
      // fp32x3: this layer's maps into the scratch with the split probability kernel (padded query rows zeroed, as
      // the forward writes them), then contact_accumulate_kernel, as ContactPredictionHead.forward runs it on the stack
      rc = attention_block(L, *wm, x, B * T, T, rope_cos, rope_sin, L->q_scale, ws, am, st, [&] {
        const size_t lbh = (size_t)i * B * H;
        int r = run_attention(ws.qkv, ws.ctx, static_cast<float*>(scratch), 0, 1, ws.as, B, T, H, st, true, nullptr,
                              L->slots);
        if (!r)
          r = run_contact_accumulate(static_cast<const float*>(scratch), (long long)H * T * T, cl.w, contact->keep,
                                     contact->acc, contact->row_part + lbh * S,
                                     contact->col_part + lbh * ((S + 15) / 16) * S, B, H, T, contact->lo, S, st);
        return r;
      });
    } else {
      rc = attention_block(L, *wm, x, B * T, T, rope_cos, rope_sin, L->q_scale, ws, am, st, [&] {
        // contacts_only: probs == nullptr and attn_flags bit 0 set, the store-free fused pass
        return run_attention(ws.qkv, ws.ctx, probs, attn_batch_stride, attn_flags, ws.as, B, T, H, st, split != 0,
                             contact ? &cl : nullptr, L->slots);  // multihead_attention.py:357-394
      });
    }
    if (!rc) rc = ffn_block(L, *wm, x, B * T, ws, am, st);
    if (rc) return rc;
    if (streamed) {  // fc2 was the slot's last reader: layer i + 2 may overwrite it
      CK(cudaEventRecord(wr.freed[i & 1], st));
      if (i + 2 < n_layers && (rc = wr.fetch(layers[i + 2], i + 2))) return rc;
    }
    if (repr_out && repr_out[i])
      CK(cudaMemcpyAsync(repr_out[i], x, (size_t)B * T * E * 4, cudaMemcpyDeviceToDevice, st));
  }
  return ESMB200_OK;
}

int esmb200_stack_forward(esmb200_layer* const* layers, int32_t n_layers, float* x, const uint8_t* pad_mask,
                          int32_t B, int32_t T, const float* rope_cos, const float* rope_sin,
                          float* const* repr_out, float* const* attn_out, int64_t attn_batch_stride,
                          int32_t attn_flags, const esmb200_contact_job* contact, void* workspace,
                          size_t workspace_bytes, void* stream) {
  return stack_forward_impl(layers, n_layers, x, pad_mask, B, T, rope_cos, rope_sin, repr_out, attn_out,
                            attn_batch_stride, attn_flags, contact, workspace, workspace_bytes, nullptr, 0, nullptr,
                            stream);
}

int esmb200_stack_forward_streamed(esmb200_layer* const* layers, int32_t n_layers, float* x, const uint8_t* pad_mask,
                                   int32_t B, int32_t T, const float* rope_cos, const float* rope_sin,
                                   float* const* repr_out, float* const* attn_out, int64_t attn_batch_stride,
                                   int32_t attn_flags, const esmb200_contact_job* contact, void* workspace,
                                   size_t workspace_bytes, void* ring, size_t ring_bytes, void* copy_stream,
                                   void* stream) {
  if (!ring) return fail(ESMB200_EINVAL, "null ring");
  return stack_forward_impl(layers, n_layers, x, pad_mask, B, T, rope_cos, rope_sin, repr_out, attn_out,
                            attn_batch_stride, attn_flags, contact, workspace, workspace_bytes, ring, ring_bytes,
                            copy_stream, stream);
}

int esmb200_stack_contacts_bytes(int32_t n_layers, int32_t num_heads, int32_t B, int32_t T, int32_t S,
                                 int32_t precision, size_t* row_part_bytes, size_t* col_part_bytes,
                                 size_t* scratch_bytes) {
  if (n_layers <= 0 || num_heads <= 0 || B <= 0 || T <= 0 || S <= 0 || S > T || precision < 0 || precision > 2)
    return fail(ESMB200_EINVAL, "bad shape");
  const ContactSizes c = contact_sizes(n_layers, num_heads, B, T, S, precision);
  if (row_part_bytes) *row_part_bytes = c.row_part;
  if (col_part_bytes) *col_part_bytes = c.col_part;
  if (scratch_bytes) *scratch_bytes = c.scratch;
  return ESMB200_OK;
}

int esmb200_stack_contacts(esmb200_layer* const* layers, int32_t n_layers, float* x, const uint8_t* pad_mask, int32_t B,
                           int32_t T, const float* rope_cos, const float* rope_sin, float* const* repr_out,
                           const esmb200_contact_job* contact, void* probs_scratch, size_t probs_scratch_bytes,
                           void* workspace, size_t workspace_bytes, void* ring, size_t ring_bytes, void* copy_stream,
                           void* stream) {
  return stack_forward_impl(layers, n_layers, x, pad_mask, B, T, rope_cos, rope_sin, repr_out, nullptr, 0,
                            1 /* padded query rows zero, as in ESM2.forward */, contact, workspace, workspace_bytes,
                            ring, ring_bytes, copy_stream, stream, true, probs_scratch, probs_scratch_bytes);
}

int esmb200_layer_forward(esmb200_layer* layer, float* x, const uint8_t* pad_mask, int32_t B, int32_t T,
                          const float* rope_cos, const float* rope_sin, float* attn_probs, void* workspace,
                          size_t workspace_bytes, void* stream) {
  if (!layer) return fail(ESMB200_EINVAL, "null layer");
  float* attn_arr[1] = {attn_probs};
  esmb200_layer* arr[1] = {layer};
  return esmb200_stack_forward(arr, 1, x, pad_mask, B, T, rope_cos, rope_sin, nullptr, attn_probs ? attn_arr : nullptr,
                               0, 0, nullptr, workspace, workspace_bytes, stream);
}

int esmb200_embed_tokens(const int64_t* tokens, const float* table, float* x, int32_t B, int32_t T, int32_t E,
                         int32_t padding_idx, int32_t mask_idx, int32_t token_dropout, void* stream) {
  if (!tokens || !table || !x) return fail(ESMB200_EINVAL, "null argument");
  if (B <= 0 || B > 65535 || T <= 0 || E % 4 != 0) return fail(ESMB200_EINVAL, "bad shape");
  ProfScope ps(T_EMBED, static_cast<cudaStream_t>(stream));
  int chunks = (8 * num_sms() + B - 1) / B;  // >= 8 blocks per SM over the batch, at least 4 rows per block
  if (chunks > (T + 3) / 4) chunks = (T + 3) / 4;
  if (chunks < 1) chunks = 1;
  embed_tokens_kernel<<<dim3(chunks, B), 256, 0, static_cast<cudaStream_t>(stream)>>>(tokens, table, x, T, E, padding_idx,
                                                                                     mask_idx, token_dropout);
  CK(cudaGetLastError());
  return ESMB200_OK;
}

int esmb200_esm1b_embed(const int64_t* tokens, const float* embed_table, const float* pos_table, const float* ln_weight,
                        const float* ln_bias, float eps, int32_t token_dropout, int32_t padding_idx, int32_t mask_idx,
                        float* x, int32_t B, int32_t T, int32_t E, void* stream) {
  if (!tokens || !embed_table || !pos_table || !x) return fail(ESMB200_EINVAL, "null argument");
  if ((ln_weight == nullptr) != (ln_bias == nullptr))
    return fail(ESMB200_EINVAL, "ln_weight and ln_bias must both be given or both be NULL");
  if (B <= 0 || B > 65535 || T <= 0 || T > 12288 || E <= 0 || E % 4 != 0 || E > 20 * 128)
    return fail(ESMB200_EINVAL, "bad shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(T_EMBED, st);
  int chunks = (8 * num_sms() + B - 1) / B;  // >= 8 blocks per SM over the batch, at least 8 rows (one per warp) per block
  if (chunks > (T + 7) / 8) chunks = (T + 7) / 8;
  if (chunks < (T + 8191) / 8192) chunks = (T + 8191) / 8192;  // a chunk's positions (4 bytes a row) stay within 48 KB
  if (chunks < 1) chunks = 1;
  const int rows = (T + chunks - 1) / chunks;
  const dim3 grid(chunks, B);
  const size_t smem = (size_t)rows * sizeof(int);
  if (E <= 4 * 128)
    esm1b_embed_kernel<4><<<grid, 256, smem, st>>>(tokens, embed_table, pos_table, ln_weight, ln_bias, eps, token_dropout,
                                                    padding_idx, mask_idx, x, T, E);
  else if (E <= 10 * 128)
    esm1b_embed_kernel<10><<<grid, 256, smem, st>>>(tokens, embed_table, pos_table, ln_weight, ln_bias, eps, token_dropout,
                                                     padding_idx, mask_idx, x, T, E);
  else
    esm1b_embed_kernel<20><<<grid, 256, smem, st>>>(tokens, embed_table, pos_table, ln_weight, ln_bias, eps, token_dropout,
                                                     padding_idx, mask_idx, x, T, E);
  CK(cudaGetLastError());
  return ESMB200_OK;
}

int esmb200_layernorm(const float* x, const float* weight, const float* bias, float* out, int32_t M, int32_t E,
                      float eps, void* stream) {
  if (!x || !weight || !bias || !out) return fail(ESMB200_EINVAL, "null argument");
  ProfScope ps(T_LN_F32, static_cast<cudaStream_t>(stream));
  cudaError_t e = launch_layernorm<0>(x, weight, bias, out, M, E, eps, static_cast<cudaStream_t>(stream));
  if (e != cudaSuccess) return fail_cuda(e, "layernorm");
  return ESMB200_OK;
}

int esmb200_layernorm_f16(const float* x, const float* weight, const float* bias, void* out, int32_t M, int32_t E,
                          float eps, void* stream) {
  if (!x || !weight || !bias || !out) return fail(ESMB200_EINVAL, "null argument");
  return layernorm_f16(x, weight, bias, out, M, E, eps, false, T_LN1, static_cast<cudaStream_t>(stream));
}

int esmb200_layernorm_fp8(const float* x, const float* weight, const float* bias, void* out_e4m3, float* scales,
                          int32_t M, int32_t E, float eps, void* stream) {
  if (!x || !weight || !bias || !out_e4m3 || !scales) return fail(ESMB200_EINVAL, "null argument");
  if (M <= 0 || E <= 0 || E % 4 != 0 || E > 40 * 128) return fail(ESMB200_EINVAL, "bad shape");
  return layernorm_fp8(x, weight, bias, out_e4m3, scales, M, E, eps, T_LN1, static_cast<cudaStream_t>(stream));
}

int esmb200_quantize_fp8(const float* src, void* dst_e4m3, float* scales, int32_t rows, int32_t K, int32_t block_rows,
                         void* stream) {
  if (!src || !dst_e4m3 || !scales) return fail(ESMB200_EINVAL, "null argument");
  if (rows <= 0 || K <= 0 || (block_rows != 1 && block_rows != 128) || rows / block_rows > 65535)
    return fail(ESMB200_EINVAL, "quantize_fp8 needs rows, K > 0 and block_rows 1 or 128");
  return quantize_fp8(src, static_cast<uint8_t*>(dst_e4m3), scales, rows, K, block_rows,
                      static_cast<cudaStream_t>(stream));
}

int esmb200_gemm_fp8(int32_t epilogue, const void* a, const float* a_scales, const void* w, const float* w_scales,
                     const float* bias, void* out, float* out_scales, int32_t M, int32_t N, int32_t K,
                     const float* rope_cos, const float* rope_sin, int32_t T, int32_t E, void* stream) {
  if (!a || !a_scales || !w || !w_scales || !bias || !out) return fail(ESMB200_EINVAL, "null argument");
  if (M <= 0 || N <= 0 || K <= 0 || K % 16 != 0) return fail(ESMB200_EINVAL, "fp8 gemm needs M, N > 0 and K % 16 == 0");
  if (epilogue == EPI_QKV_ROPE &&
      (N % 64 != 0 || !rope_cos || !rope_sin || T <= 0 || E <= 0 || E % 64 != 0 || N != 3 * E))
    return fail(ESMB200_EINVAL, "qkv epilogue needs rope tables, T and N == 3E, E % 64 == 0");
  if (epilogue == EPI_BIAS_RESIDUAL && N % 32 != 0) return fail(ESMB200_EINVAL, "residual epilogue needs N % 32 == 0");
  if (epilogue == EPI_GELU_FP8 && (N % 128 != 0 || !out_scales))
    return fail(ESMB200_EINVAL, "gelu -> fp8 epilogue needs N % 128 == 0 and out_scales");
  if (epilogue != EPI_QKV_ROPE && epilogue != EPI_BIAS_RESIDUAL && epilogue != EPI_GELU_FP8)
    return fail(ESMB200_EINVAL, "fp8 gemm epilogue must be 0 (qkv), 1 (residual) or 5 (gelu -> fp8)");
  int rc = check_device();
  if (rc) return rc;
  CUtensorMap ta, tb, to;
  rc = make_tmap_2d(&ta, a, 1, M, K, K, gemm_fp8_cfg::BOX_ROWS);
  if (!rc) rc = make_tmap_2d(&tb, w, 1, N, K, K, gemm_fp8_cfg::BOX_ROWS);
  if (!rc) rc = make_gemm_out_map(&to, out, epilogue == EPI_QKV_ROPE ? 2 : epilogue == EPI_GELU_FP8 ? 1 : 4, M, N);
  if (rc) return rc;
  GemmParams g = gemm_params(M, N, K, bias);
  g.rope_cos = rope_cos; g.rope_sin = rope_sin; g.T = T; g.E = E; g.q_scale = 0.125f;
  return launch_gemm_fp8(epilogue, ta, tb, to, {g, a_scales, w_scales, out_scales}, static_cast<cudaStream_t>(stream));
}

int esmb200_gemm_f16(int32_t epilogue, const void* a, const void* w, const float* bias, void* out, int32_t M,
                     int32_t N, int32_t K, const float* rope_cos, const float* rope_sin, int32_t T, int32_t E,
                     void* stream) {
  return gemm_epilogue_entry(epilogue, a, w, bias, out, M, N, K, rope_cos, rope_sin, T, E, false, stream);
}

// ---- fp32x3 precision building blocks (hi | lo fp16 operands): used by the LM head, the MSA layer's attention-map path
// and the kernel-level parity tests
int esmb200_layernorm_split(const float* x, const float* weight, const float* bias, void* out, int32_t M, int32_t E,
                            float eps, void* stream) {
  if (!x || !weight || !bias || !out) return fail(ESMB200_EINVAL, "null argument");
  return layernorm_f16(x, weight, bias, out, M, E, eps, true, T_LN1, static_cast<cudaStream_t>(stream));
}

int esmb200_convert_split(const float* src, void* dst, int64_t rows, int32_t K, void* stream) {
  if (!src || !dst) return fail(ESMB200_EINVAL, "null argument");
  if (rows <= 0 || K <= 0) return ESMB200_OK;
  return convert_f16(src, dst, (size_t)rows, K, true, static_cast<cudaStream_t>(stream));
}

int esmb200_gemm_split(int32_t epilogue, const void* a, const void* w, const float* bias, void* out, int32_t M,
                       int32_t N, int32_t K, const float* rope_cos, const float* rope_sin, int32_t T, int32_t E,
                       void* stream) {
  return gemm_epilogue_entry(epilogue, a, w, bias, out, M, N, K, rope_cos, rope_sin, T, E, true, stream);
}

int esmb200_attention_split(const void* qkv, const uint8_t* pad_mask, void* ctx, float* attn_probs, int32_t B, int32_t T,
                            int32_t H, void* scratch, void* stream) {
  return attention_entry(qkv, pad_mask, ctx, attn_probs, B, T, H, scratch, stream, true, 1);
}

int esmb200_gemm_qkv_f16(const void* a, const void* w, const float* bias, void* out, int32_t M, int32_t E, float q_scale,
                         const float* rope_cos, const float* rope_sin, int32_t T, void* stream) {
  if (!a || !w || !bias || !out) return fail(ESMB200_EINVAL, "null argument");
  if (M <= 0 || E <= 0 || E % 64 != 0) return fail(ESMB200_EINVAL, "qkv gemm needs E % 64 == 0");
  if ((rope_cos == nullptr) != (rope_sin == nullptr) || (rope_cos && T <= 0))
    return fail(ESMB200_EINVAL, "rope tables must be given together with T, or not at all");
  int rc = check_device();
  if (rc) return rc;
  return run_gemm(EPI_QKV_ROPE, a, w, bias, out, M, 3 * E, E, rope_cos, rope_sin, T > 0 ? T : 1, E, q_scale, false,
                  stream);
}

int esmb200_gemm_qkv_split(const void* a, const void* w, const float* bias, void* out, int32_t M, int32_t E,
                           float q_scale, void* stream) {
  if (!a || !w || !bias || !out) return fail(ESMB200_EINVAL, "null argument");
  if (M <= 0 || E <= 0 || E % 64 != 0) return fail(ESMB200_EINVAL, "qkv gemm needs E % 64 == 0");
  int rc = check_device();
  if (rc) return rc;
  return run_gemm(EPI_QKV_ROPE, a, w, bias, out, M, 3 * E, E, nullptr, nullptr, 1, E, q_scale, true, stream);
}

int esmb200_gemm_qkv_heads(int32_t precision, const void* a, const float* a_scales, const void* w,
                           const float* w_scales, const float* bias, void* out, int32_t M, int32_t E, int32_t H,
                           float q_scale, const float* rope_cos, const float* rope_sin, int32_t T, void* stream) {
  if (!a || !w || !bias || !out) return fail(ESMB200_EINVAL, "null argument");
  if (precision < 0 || precision > 2) return fail(ESMB200_EINVAL, "precision must be 0 (fp16), 1 (fp32x3) or 2 (fp8)");
  if (precision == 2 && (!a_scales || !w_scales))
    return fail(ESMB200_EINVAL, "fp8 precision needs a_scales and w_scales");
  // the shapes esmb200_layer_create refuses, with its messages
  if (M <= 0 || E <= 0 || H <= 0 || E % H != 0)
    return fail(ESMB200_EINVAL, "embed_dim must be a positive multiple of num_heads");
  const int d = E / H;
  if (d > 128 || d % 2 != 0)
    return fail(ESMB200_EINVAL, "esmb200 supports even head_dim <= 128 (every ESM-2 model, MSA Transformer)");
  if (E % 16 != 0) return fail(ESMB200_EINVAL, "embed_dim must be a multiple of 16");
  const int slots = head_slots(E, H);
  if (precision == 1 && slots == 2) return fail(ESMB200_EINVAL, "fp32x3 precision is not available for head_dim > 64");
  if (precision == 1 && E % 64 != 0)
    return fail(ESMB200_EINVAL, "fp32x3 precision needs embed_dim % 64 == 0 (all ESM-2 models except 35M)");
  if ((rope_cos == nullptr) != (rope_sin == nullptr) || (rope_cos && T <= 0))
    return fail(ESMB200_EINVAL, "rope tables must be given together with T, or not at all");
  int rc = check_device();
  if (rc) return rc;
  const int Ea = 64 * slots * H;
  const GemmParams g = qkv_params(M, E, Ea, slots, bias, rope_cos, rope_sin, T > 0 ? T : 1, q_scale);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  CUtensorMap ta, tb, to;
  if (precision == 2) {
    rc = make_tmap_2d(&ta, a, 1, M, E, E, gemm_fp8_cfg::BOX_ROWS);
    if (!rc) rc = make_tmap_2d(&tb, w, 1, 3 * (uint64_t)Ea, E, E, gemm_fp8_cfg::BOX_ROWS);
    if (!rc) rc = make_gemm_out_map(&to, out, 2, M, 3 * (uint64_t)Ea);
    return rc ? rc : launch_gemm_fp8(EPI_QKV_ROPE, ta, tb, to, {g, a_scales, w_scales, nullptr}, st);
  }
  const uint64_t pf = precision == 1 ? 2 : 1;
  rc = make_tmap_f16(&ta, a, M, pf * E, pf * E, gemm2_cfg::BOX_M);
  if (!rc) rc = make_tmap_f16(&tb, w, 3 * (uint64_t)Ea, pf * E, pf * E, gemm2_cfg::HALF_N);
  if (!rc) rc = make_gemm_out_map(&to, out, 2, M, pf * 3 * Ea);
  return rc ? rc : launch_gemm(EPI_QKV_ROPE, ta, tb, to, g, st, T_GEMM_OTHER, precision == 1);
}

int esmb200_attention(const void* qkv, const uint8_t* pad_mask, void* ctx, float* attn_probs, int32_t B, int32_t T,
                      int32_t H, void* scratch, void* stream) {
  return attention_entry(qkv, pad_mask, ctx, attn_probs, B, T, H, scratch, stream, false, 1);
}

int esmb200_attention128(const void* qkv, const uint8_t* pad_mask, void* ctx, float* attn_probs, int32_t B, int32_t T,
                         int32_t H, void* scratch, void* stream) {
  return attention_entry(qkv, pad_mask, ctx, attn_probs, B, T, H, scratch, stream, false, 2);
}

// ---- MSA axial attention (esm/axial_attention.py) -----------------------------------------------------------------
size_t esmb200_tied_row_attention_scratch_bytes(int32_t B, int32_t C, int32_t H) {
  return tied_scratch_bytes(B, C, H, 0);
}

size_t esmb200_tied_row_attention_split_scratch_bytes(int32_t B, int32_t C, int32_t H) {
  return tied_scratch_bytes(B, C, H, 1);
}

static int tied_row_impl(const void* qkv, const uint8_t* key_pad, long long key_pad_stride, void* ctx,
                         float* attn_probs, int32_t B, int32_t R, int32_t C, int32_t H, void* scratch,
                         size_t scratch_bytes, void* stream, bool split = false) {
  if (!qkv || !ctx || !scratch) return fail(ESMB200_EINVAL, "null argument");
  if (B <= 0 || R <= 0 || C <= 0 || H <= 0 || H > 64 || (long long)B * H > 65535)
    return fail(ESMB200_EINVAL, "bad shape");
  if (C > TIED_MAX_C) return fail(ESMB200_EINVAL, "tied row attention supports at most 1024 alignment columns");
  if (scratch_bytes < tied_scratch_bytes(B, C, H, split))
    return fail(ESMB200_EWORKSPACE, "tied row attention scratch too small");
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int E = H * 64;
  const size_t Cp = align_up((size_t)C, 64);
  uint8_t* sp = reinterpret_cast<uint8_t*>(align_up(reinterpret_cast<uintptr_t>(scratch), 1024));
  TiedParams tp;
  tp.B = B; tp.R = R; tp.C = C; tp.H = H; tp.E = E; tp.Cp = (int)Cp;
  tp.S = attn_probs ? attn_probs : reinterpret_cast<float*>(sp);
  tp.P = reinterpret_cast<__half*>(sp + align_up((size_t)H * B * C * C * 4, 1024));  // [H*B*C, Cp] (split: 2*Cp)
  tp.ctx = static_cast<__half*>(ctx);
  tp.key_pad = key_pad;
  tp.key_pad_stride = key_pad_stride;
  tp.write_probs = attn_probs ? 1 : 0;
  const uint64_t rows = (uint64_t)B * R * C;
  const uint64_t qcols = (uint64_t)(split ? 6 : 3) * E, pcols = (split ? 2 : 1) * Cp;  // split: hi | lo
  CUtensorMap tq, tk, tv, tpm;
  if ((rc = make_tmap_f16(&tq, qkv, rows, qcols, qcols, tied_cfg::S_BM))) return rc;
  if ((rc = make_tmap_f16(&tk, qkv, rows, qcols, qcols, tied_cfg::S_BN))) return rc;
  if ((rc = make_tmap_f16(&tv, qkv, rows, qcols, qcols, 64))) return rc;
  if ((rc = make_tmap_f16(&tpm, tp.P, (uint64_t)H * B * C, pcols, pcols, tied_cfg::V_BM))) return rc;
  cudaError_t e;
  {
    ProfScope ps(T_TIED_SCORES, st);
    e = split ? launch_tied_scores<true>(tq, tk, tp, st) : launch_tied_scores<false>(tq, tk, tp, st);
  }
  if (e != cudaSuccess) return fail_cuda(e, "tied scores launch");
  {
    ProfScope ps(T_TIED_SOFTMAX, st);
    e = split ? launch_tied_softmax<true>(tp, st) : launch_tied_softmax<false>(tp, st);
  }
  if (e != cudaSuccess) return fail_cuda(e, "tied softmax launch");
  {
    ProfScope ps(T_TIED_PV, st);
    e = split ? launch_tied_pv<true>(tpm, tv, tp, st) : launch_tied_pv<false>(tpm, tv, tp, st);
  }
  if (e != cudaSuccess) return fail_cuda(e, "tied update launch");
  return ESMB200_OK;
}

int esmb200_tied_row_attention(const void* qkv, const uint8_t* key_pad, void* ctx, float* attn_probs, int32_t B,
                               int32_t R, int32_t C, int32_t H, void* scratch, size_t scratch_bytes, void* stream) {
  return tied_row_impl(qkv, key_pad, C, ctx, attn_probs, B, R, C, H, scratch, scratch_bytes, stream);
}

int esmb200_tied_row_attention_split(const void* qkv, const uint8_t* key_pad, void* ctx, float* attn_probs, int32_t B,
                                     int32_t R, int32_t C, int32_t H, void* scratch, size_t scratch_bytes,
                                     void* stream) {
  return tied_row_impl(qkv, key_pad, C, ctx, attn_probs, B, R, C, H, scratch, scratch_bytes, stream, true);
}

static int column_entry(const void* qkv, const uint8_t* pad_mask, void* ctx, int32_t B, int32_t R, int32_t C,
                        int32_t H, void* scratch, void* stream, bool split) {
  if (!qkv || !ctx || !scratch) return fail(ESMB200_EINVAL, "null argument");
  if (B <= 0 || R <= 0 || C <= 0 || H <= 0 || H > 64) return fail(ESMB200_EINVAL, "bad shape");
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const AttnScratch s = attn_scratch_layout(reinterpret_cast<uintptr_t>(scratch), B * C, R, H);
  rc = run_key_bits(pad_mask, s, B * C, R, st);
  if (rc) return rc;
  return run_column_attention(qkv, ctx, s, B, R, C, H, st, split);
}

int esmb200_column_attention(const void* qkv, const uint8_t* pad_mask, void* ctx, int32_t B, int32_t R, int32_t C,
                             int32_t H, void* scratch, void* stream) {
  return column_entry(qkv, pad_mask, ctx, B, R, C, H, scratch, stream, false);
}

int esmb200_column_attention_split(const void* qkv, const uint8_t* pad_mask, void* ctx, int32_t B, int32_t R, int32_t C,
                                   int32_t H, void* scratch, void* stream) {
  return column_entry(qkv, pad_mask, ctx, B, R, C, H, scratch, stream, true);
}

size_t esmb200_axial_workspace_bytes(int32_t E, int32_t F, int32_t B, int32_t R, int32_t C) {
  return axial_workspace_layout(nullptr, E, F, B, R, C, 0).bytes;
}

size_t esmb200_axial_workspace_bytes_split(int32_t E, int32_t F, int32_t B, int32_t R, int32_t C) {
  return axial_workspace_layout(nullptr, E, F, B, R, C, 1).bytes;
}

// (A CUDA-graph replay of this launch sequence was measured: 20.70 vs 20.77 ms per 128 x 512 MSA — the ~2 ms between the
// sum of the kernel times and the wall time are not host launch overhead, so the calls stay plain stream launches.)
int esmb200_axial_stack_forward(esmb200_layer* const* row_layers, esmb200_layer* const* col_layers, int32_t n_layers,
                                float* x, const uint8_t* pad_mask, const uint8_t* col_pad_mask, int32_t B, int32_t R,
                                int32_t C, float* const* row_attn_out, float* const* col_attn_out, void* workspace,
                                size_t workspace_bytes, void* stream) {
  if (!row_layers || !col_layers || n_layers <= 0 || !x || !workspace) return fail(ESMB200_EINVAL, "null argument");
  if (B <= 0 || R <= 0 || C <= 0) return fail(ESMB200_EINVAL, "empty alignment");
  if ((pad_mask == nullptr) != (col_pad_mask == nullptr))
    return fail(ESMB200_EINVAL, "pad_mask [B,R,C] and col_pad_mask [B,C,R] must be given together");
  if ((long long)B * R * C > 0x7fffffffLL / 8) return fail(ESMB200_EINVAL, "B*R*C too large for one call");
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int i = 0; i < n_layers; ++i)
    if ((row_layers[i] && row_layers[i]->fp8) || (col_layers[i] && col_layers[i]->fp8))
      return fail(ESMB200_EINVAL, "the MSA axial stack runs fp16 or fp32x3 layers, not fp8");
  const int E = col_layers[0]->E, F = col_layers[0]->F, H = col_layers[0]->H;
  if (F <= 0) return fail(ESMB200_EINVAL, "col_layers carry the feed-forward weights");
  const int split = col_layers[0]->split;
  for (int i = 0; i < n_layers; ++i)
    if (row_layers[i]->E != E || col_layers[i]->E != E || col_layers[i]->F != F || row_layers[i]->H != H ||
        col_layers[i]->H != H)
      return fail(ESMB200_EINVAL, "layers of one stack must share E, H and F");
  for (int i = 0; i < n_layers; ++i)
    if (row_layers[i]->split != split || col_layers[i]->split != split)
      return fail(ESMB200_EINVAL, "the row and column layers of one stack must share one precision");
  for (int i = 0; i < n_layers; ++i)
    if (col_layers[i]->host)
      return fail(ESMB200_EINVAL, "col layer " + std::to_string(i) + " is offloaded to host memory: the MSA axial "
                                  "stack runs resident layers only");
  const AxialWorkspace aw = axial_workspace_layout(workspace, E, F, B, R, C, split);
  if (workspace_bytes < aw.bytes) return fail(ESMB200_EWORKSPACE, "workspace too small");
  if (E != 64 * H) return fail(ESMB200_EINVAL, "the MSA axial path needs head_dim 64");
  const int M = B * R * C;
  const Workspace& ws = aw.ws;
  ActMaps am;
  rc = make_act_maps(&am, ws, x, E, H, F, M, split);
  if (rc) return rc;
  rc = run_key_bits(col_pad_mask, ws.as, B * C, R, st);  // column attention: B*C sequences of R keys
  if (rc) return rc;
  // axial_attention.py:36-38: scaling / math.sqrt(num_rows) in double, rounded to fp32 by `q *= ...` (0.125f /
  // sqrtf(R) in fp32 is one ulp off at 242 of the depths R = 1 ... 1024, the first R = 6, 7 and 17)
  const float row_scale = (float)(pow(64.0, -0.5) / sqrt((double)R));
  for (int i = 0; i < n_layers; ++i) {
    // tied row attention (modules.py:202-207; axial_attention.py:71-130)
    rc = attention_block(row_layers[i], row_layers[i]->tm, x, M, 1, nullptr, nullptr, row_scale, ws, am, st, [&]() -> int {
      if (pad_mask) {
        ProfScope ps(T_KEYBITS, st);
        if (split)
          zero_q_at_pads_kernel<true><<<(M + 7) / 8, 256, 0, st>>>(ws.qkv, pad_mask, M, E);
        else
          zero_q_at_pads_kernel<false><<<(M + 7) / 8, 256, 0, st>>>(ws.qkv, pad_mask, M, E);
        CK(cudaGetLastError());
      }
      return tied_row_impl(ws.qkv, pad_mask, (long long)R * C, ws.ctx, row_attn_out ? row_attn_out[i] : nullptr, B, R,
                           C, H, aw.tied, aw.tied_bytes, stream, split != 0);
    });
    // column attention (modules.py:208-212; axial_attention.py:182-239)
    if (!rc)
      rc = attention_block(col_layers[i], col_layers[i]->tm, x, M, 1, nullptr, nullptr, col_layers[i]->q_scale, ws, am,
                           st, [&] {
                             return run_column_attention(ws.qkv, ws.ctx, ws.as, B, R, C, H, st, split != 0,
                                                         col_attn_out ? col_attn_out[i] : nullptr);
                           });
    // feed-forward (modules.py:213-214)
    if (!rc) rc = ffn_block(col_layers[i], col_layers[i]->tm, x, M, ws, am, st);
    if (rc) return rc;
  }
  return ESMB200_OK;
}

int esmb200_msa_embed(const int64_t* tokens, const float* embed_table, const float* pos_table, const float* msa_pos,
                      int32_t msa_pos_dim, const float* ln_weight, const float* ln_bias, float eps, float* x,
                      int32_t B, int32_t R, int32_t C, int32_t E, int32_t padding_idx, void* stream) {
  if (!tokens || !embed_table || !pos_table || !ln_weight || !ln_bias || !x) return fail(ESMB200_EINVAL, "null argument");
  // C <= 12288: a row's positions (4 bytes a column) are held in 48 KB of shared memory
  if (B <= 0 || R <= 0 || C <= 0 || C > 12288 || E <= 0 || E % 4 != 0 || E > 20 * 128)
    return fail(ESMB200_EINVAL, "bad shape");
  if (msa_pos && msa_pos_dim != E && msa_pos_dim != 1)
    return fail(ESMB200_EINVAL, "msa_position_embedding width must be E or 1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(T_EMBED, st);
  const size_t smem = (size_t)C * sizeof(int);
  const int grid = B * R;
  if (E <= 4 * 128)
    msa_embed_kernel<4><<<grid, 256, smem, st>>>(tokens, embed_table, pos_table, msa_pos, msa_pos_dim, ln_weight,
                                                  ln_bias, eps, x, R, C, E, padding_idx);
  else if (E <= 10 * 128)
    msa_embed_kernel<10><<<grid, 256, smem, st>>>(tokens, embed_table, pos_table, msa_pos, msa_pos_dim, ln_weight,
                                                   ln_bias, eps, x, R, C, E, padding_idx);
  else
    msa_embed_kernel<20><<<grid, 256, smem, st>>>(tokens, embed_table, pos_table, msa_pos, msa_pos_dim, ln_weight,
                                                   ln_bias, eps, x, R, C, E, padding_idx);
  CK(cudaGetLastError());
  return ESMB200_OK;
}


int esmb200_contact_accumulate(const float* attn, int64_t batch_stride, const float* w, const uint8_t* keep, float* acc,
                               float* row_sum, float* col_part, int32_t B, int32_t H, int32_t T, int32_t lo, int32_t hi,
                               void* stream) {
  if (!attn || !w || !acc || !row_sum || !col_part) return fail(ESMB200_EINVAL, "null argument");
  const int S = hi - lo;
  if (B <= 0 || H <= 0 || T <= 0 || lo < 0 || hi > T || S <= 0 || B > 65535) return fail(ESMB200_EINVAL, "bad shape");
  if (S > kContactMaxS) return fail(ESMB200_EINVAL, kContactMaxSMsg);
  return run_contact_accumulate(attn, batch_stride, w, keep, acc, row_sum, col_part, B, H, T, lo, S,
                                static_cast<cudaStream_t>(stream));
}

int esmb200_contact_finalize(const float* acc, const float* u, const float* a1, const float* bias, float* out, int32_t B,
                             int32_t C, int32_t S, void* stream) {
  if (!acc || !u || !a1 || !out) return fail(ESMB200_EINVAL, "null argument");
  if (B <= 0 || C <= 0 || S <= 0 || B > 65535) return fail(ESMB200_EINVAL, "bad shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(T_PROBS, st);
  dim3 grid((S + 63) / 64, (S + 63) / 64, B);
  contact_finalize_kernel<<<grid, 256, 0, st>>>(acc, u, a1, bias, out, C, S);
  CK(cudaGetLastError());
  return ESMB200_OK;
}


int esmb200_mean_pool(const float* x, const int32_t* lengths, float* out, int32_t B, int32_t T, int32_t E,
                      void* stream) {
  if (!x || !lengths || !out) return fail(ESMB200_EINVAL, "null argument");
  if (B <= 0 || T < 2 || E <= 0 || B > 65535) return fail(ESMB200_EINVAL, "bad shape");
  if (E % 4 != 0) return fail(ESMB200_EINVAL, "mean_pool needs E % 4 == 0");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(T_MEANPOOL, st);
  dim3 grid((E + 127) / 128, B);
  mean_pool_kernel<<<grid, 256, 0, st>>>(x, lengths, out, T, E);
  CK(cudaGetLastError());
  return ESMB200_OK;
}

int esmb200_log_softmax_rows(const float* logits, int64_t ld, int32_t n, int32_t V, const int64_t* target, float* out,
                             void* stream) {
  if (!logits || !out) return fail(ESMB200_EINVAL, "null argument");
  if (n < 0 || V <= 0 || V > 64 || ld < V) return fail(ESMB200_EINVAL, "log_softmax_rows needs 0 < V <= 64 and ld >= V");
  if (n == 0) return ESMB200_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(T_LOG_SOFTMAX, st);
  log_softmax_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(logits, ld, n, V, target, out);
  CK(cudaGetLastError());
  return ESMB200_OK;
}


int esmb200_window_merge(const float* src, int64_t src_ld, const int64_t* idx, const float* w, const int64_t* seg,
                         int32_t rows, int32_t C, float* out, int64_t out_ld, void* stream) {
  if (rows < 0 || C <= 0 || src_ld < C || out_ld < C)
    return fail(ESMB200_EINVAL, "window_merge needs rows >= 0, C > 0, src_ld >= C and out_ld >= C");
  if (rows == 0) return ESMB200_OK;
  if (!src || !idx || !w || !seg || !out) return fail(ESMB200_EINVAL, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(T_WINDOW_MERGE, st);
  const int64_t total = (int64_t)rows * C;
  const int64_t blocks = (total + 255) / 256;
  window_merge_kernel<<<(unsigned)(blocks < 65536 ? blocks : 65536), 256, 0, st>>>(src, src_ld, idx, w, seg, rows, C,
                                                                                  out, out_ld);
  CK(cudaGetLastError());
  return ESMB200_OK;
}


size_t esmb200_jacobian_scratch_bytes(int32_t L) { return L < 2 ? 0 : jacobian_scratch(nullptr, L).bytes; }

int esmb200_jacobian_contacts(const float* jac, int32_t L, void* scratch, size_t scratch_bytes, float* contacts,
                              void* stream) {
  if (L < 2 || L > 65535) return fail(ESMB200_EINVAL, "jacobian_contacts needs 2 <= L <= 65535");
  if (!jac || !scratch || !contacts) return fail(ESMB200_EINVAL, "null argument");
  const JacobianScratch s = jacobian_scratch(static_cast<char*>(scratch), L);
  if (scratch_bytes < s.bytes) return fail(ESMB200_EINVAL, "scratch smaller than esmb200_jacobian_scratch_bytes(L)");
  if (reinterpret_cast<uintptr_t>(scratch) % 256 != 0) return fail(ESMB200_EINVAL, "scratch must be 256-byte aligned");
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned tiles = (unsigned)((L + kJacTileJ - 1) / kJacTileJ);
  {  // one ProfScope per kernel: esmb200_launch_count counts kernels
    ProfScope ps(T_JACOBIAN, st);
    jacobian_marginals_kernel<<<dim3(tiles, kJacAA), 320, 0, st>>>(jac, L, s.s_i, s.part);
    CK(cudaGetLastError());
  }
  {
    ProfScope ps(T_JACOBIAN, st);
    const size_t n = (size_t)L * kJacAA * kJacAA + kJacAA * kJacAA;
    jacobian_finish_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s.s_i, s.part, L, s.s_j, s.s);
    CK(cudaGetLastError());
  }
  {
    ProfScope ps(T_JACOBIAN, st);
    const dim3 grid((unsigned)((L + kJacNormJ - 1) / kJacNormJ), (unsigned)L);
    jacobian_norms_kernel<<<grid, kJacNormJ * kJacAA, 0, st>>>(jac, s.s_i, s.s_j, s.s, L, s.n);
    CK(cudaGetLastError());
  }
  {
    ProfScope ps(T_JACOBIAN, st);
    jacobian_apc_sums_kernel<<<(unsigned)((L + 255) / 256 + (L + 7) / 8), 256, 0, st>>>(s.n, L, s.row, s.col);
    CK(cudaGetLastError());
  }
  {
    ProfScope ps(T_JACOBIAN, st);
    const size_t blocks = ((size_t)L * L + 255) / 256;
    jacobian_apc_kernel<<<(unsigned)(blocks < 1024 ? blocks : 1024), 256, 0, st>>>(s.n, s.row, s.col, L, contacts);
    CK(cudaGetLastError());
  }
  return ESMB200_OK;
}


int esmb200_sample_order(const int64_t* entries, int32_t n, int32_t n_chains, int64_t chain0, int64_t sweep,
                         uint64_t seed, int64_t* keys, void* stream) {
  if (n <= 0 || n_chains < 0) return fail(ESMB200_EINVAL, "sample_order needs n > 0 and n_chains >= 0");
  if (chain0 < 0 || chain0 + n_chains > (int64_t(1) << 32) || sweep < 0 || sweep >= (int64_t(1) << 32))
    return fail(ESMB200_EINVAL, "sample_order needs chain0 + n_chains <= 2^32 and 0 <= sweep < 2^32");
  if (n_chains == 0) return ESMB200_OK;
  if (!entries || !keys) return fail(ESMB200_EINVAL, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ProfScope ps(T_SAMPLING, st);
  const int64_t total = (int64_t)n * n_chains;
  const int64_t blocks = (total + 255) / 256;
  sample_order_kernel<<<(unsigned)(blocks < 65536 ? blocks : 65536), 256, 0, st>>>(entries, n, total,
                                                                                  (uint32_t)chain0, (uint32_t)sweep,
                                                                                  seed, keys);
  CK(cudaGetLastError());
  return ESMB200_OK;
}

int esmb200_sample_rows(const float* logits, int64_t ld, int32_t n, const int32_t* token_set, int32_t n_tokens,
                        float temperature, uint64_t seed, int64_t step, int64_t chain0, int32_t per_chain,
                        const int64_t* entries, int64_t* tokens, int64_t chain_stride, int32_t R, int32_t C,
                        float* logq, float* logp, int64_t logp_stride, void* stream) {
  if (n < 0 || per_chain <= 0 || n % per_chain != 0)
    return fail(ESMB200_EINVAL, "sample_rows needs n >= 0 and per_chain > 0 dividing n");
  if (n_tokens < 1 || n_tokens > 32 || ld < 1)
    return fail(ESMB200_EINVAL, "sample_rows needs 1 <= n_tokens <= 32 and ld >= 1");
  if (!(temperature > 0.f) || !(temperature < INFINITY))
    return fail(ESMB200_EINVAL, "sample_rows needs a finite temperature > 0");
  if (R < 1 || C < 2 || chain_stride < (int64_t)R * C)
    return fail(ESMB200_EINVAL, "sample_rows needs R >= 1, C >= 2 and chain_stride >= R * C");
  const int64_t n_chains = n / per_chain;
  if (chain0 < 0 || chain0 + n_chains > (int64_t(1) << 32) || step < 0 || step >= (int64_t(1) << 32))
    return fail(ESMB200_EINVAL, "sample_rows needs chain0 + n / per_chain <= 2^32 and 0 <= step < 2^32");
  if (logp && logp_stride < 1) return fail(ESMB200_EINVAL, "sample_rows needs logp_stride >= 1");
  if (n == 0) return ESMB200_OK;
  if (!logits || !token_set || !entries || !tokens || !logq) return fail(ESMB200_EINVAL, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  {  // one ProfScope per kernel: esmb200_launch_count counts kernels
    ProfScope ps(T_SAMPLING, st);
    sample_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(logits, ld, n, token_set, n_tokens, temperature, seed,
                                                                (uint32_t)step, (uint32_t)chain0, per_chain, entries,
                                                                tokens, chain_stride, R, C, logq);
    CK(cudaGetLastError());
  }
  if (logp) {
    ProfScope ps(T_SAMPLING, st);
    sample_logp_kernel<<<(unsigned)((n_chains + 255) / 256), 256, 0, st>>>(logq, n_chains, per_chain, logp,
                                                                           logp_stride);
    CK(cudaGetLastError());
  }
  return ESMB200_OK;
}


size_t esmb200_msa_select_scratch_bytes(int32_t N, int32_t C, int32_t k) {
  if (N < 0 || C < 0 || k < 0) return 0;
  return msa_select_scratch(nullptr, N, C, k).bytes;
}

int esmb200_msa_greedy_select(const uint8_t* rows, int64_t ld, int32_t N, int32_t C, int32_t k, int32_t mode,
                              int64_t* selected, void* scratch, size_t scratch_bytes, void* stream) {
  if (C < 1 || C > 65535) return fail(ESMB200_EINVAL, "msa_greedy_select needs 1 <= C <= 65535");
  if (N < 0 || k < 0 || k > N) return fail(ESMB200_EINVAL, "msa_greedy_select needs 0 <= k <= N");
  if (mode != ESMB200_SELECT_MAX && mode != ESMB200_SELECT_MIN)
    return fail(ESMB200_EINVAL, "msa_greedy_select mode must be ESMB200_SELECT_MAX or ESMB200_SELECT_MIN");
  if (ld < C || ld % 16 != 0) return fail(ESMB200_EINVAL, "msa_greedy_select needs ld >= C and ld % 16 == 0");
  if (k == 0) return ESMB200_OK;
  if (!rows || !selected || !scratch) return fail(ESMB200_EINVAL, "null argument");
  if (reinterpret_cast<uintptr_t>(rows) % 16 != 0) return fail(ESMB200_EINVAL, "rows must be 16-byte aligned");
  const MsaSelectScratch s = msa_select_scratch(static_cast<char*>(scratch), N, C, k);
  if (scratch_bytes < s.bytes) return fail(ESMB200_EINVAL, "scratch smaller than esmb200_msa_select_scratch_bytes");
  if (reinterpret_cast<uintptr_t>(scratch) % 256 != 0) return fail(ESMB200_EINVAL, "scratch must be 256-byte aligned");
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)ld;
  if (smem > 48 * 1024) {  // the picked row: C <= 65535, so at most 64 KiB
    CK(cudaFuncSetAttribute(msa_select_step_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(msa_select_step_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  {  // one ProfScope per kernel: esmb200_launch_count counts kernels
    ProfScope ps(T_MSA_SELECT, st);
    const int n = N > C + 1 ? N : C + 1;
    msa_select_init_kernel<<<(unsigned)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024), 256, 0, st>>>(
        N, C, s.dist, s.picked, s.ticket, selected);
    CK(cudaGetLastError());
  }
  const unsigned blocks = (unsigned)(((int64_t)N + kSelThreads - 1) / kSelThreads);
  for (int t = 1; t < k; ++t) {  // the picked index stays on the device: no host synchronisation in this loop
    ProfScope ps(T_MSA_SELECT, st);
    if (mode == ESMB200_SELECT_MAX)
      msa_select_step_kernel<true><<<blocks, kSelThreads, smem, st>>>(rows, ld, N, t, selected, s);
    else
      msa_select_step_kernel<false><<<blocks, kSelThreads, smem, st>>>(rows, ld, N, t, selected, s);
    CK(cudaGetLastError());
  }
  return ESMB200_OK;
}


extern "C++" {
namespace {
// the fused GEMM + top-k launch both search calls share
template <bool STREAM>
int knn_launch_topk(const CUtensorMap& tq, const CUtensorMap& tx, const KnnParams& p, int splits, cudaStream_t st) {
  CK(cudaFuncSetAttribute(knn_topk_kernel<STREAM>, cudaFuncAttributeMaxDynamicSharedMemorySize, knn_cfg::SMEM_BYTES));
  ProfScope ps(T_KNN, st);  // one ProfScope per kernel: esmb200_launch_count counts kernels
  const int64_t grid = (int64_t)p.query_blocks * splits;
  knn_topk_kernel<STREAM><<<(unsigned)grid, knn_cfg::NUM_THREADS, knn_cfg::SMEM_BYTES, st>>>(tq, tx, p);
  CK(cudaGetLastError());
  return ESMB200_OK;
}
}  // namespace
}  // extern "C++"

int esmb200_knn_scratch_bytes(int32_t Q, int32_t k, int32_t splits, size_t* out) {
  if (!out) return fail(ESMB200_EINVAL, "null argument");
  if (Q < 0 || k < 1 || k > knn_cfg::MAX_K || splits < 1 || splits > knn_cfg::MAX_SPLITS)
    return fail(ESMB200_EINVAL, "knn_scratch_bytes needs Q >= 0, 1 <= k <= 128 and 1 <= splits <= 1024");
  *out = (size_t)splits * (size_t)Q * (size_t)k * 8;
  return ESMB200_OK;
}

int esmb200_knn_search(const void* queries, int64_t q_ld, int32_t Q, const void* base, int64_t b_ld, int64_t N,
                       int32_t D, const float* beta, float alpha, int64_t self_offset, int32_t k, int32_t splits,
                       void* scratch, size_t scratch_bytes, float* out_scores, int64_t* out_idx, void* stream) {
  if (k < 1 || k > knn_cfg::MAX_K) return fail(ESMB200_EINVAL, "knn_search needs 1 <= k <= 128");
  if (Q < 0 || N < 1 || N > INT32_MAX) return fail(ESMB200_EINVAL, "knn_search needs Q >= 0 and 1 <= N < 2^31");
  if (k > (self_offset >= 0 ? N - 1 : N))
    return fail(ESMB200_EINVAL, "knn_search needs k <= N candidates (N - 1 with self_offset >= 0)");
  if (D < 64 || D % 64 != 0) return fail(ESMB200_EINVAL, "knn_search needs D % 64 == 0");
  if (q_ld < D || b_ld < D || q_ld % 8 != 0 || b_ld % 8 != 0)
    return fail(ESMB200_EINVAL, "knn_search needs q_ld, b_ld >= D and multiples of 8 (16-byte rows for TMA)");
  if (splits < 1 || splits > knn_cfg::MAX_SPLITS) return fail(ESMB200_EINVAL, "knn_search needs 1 <= splits <= 1024");
  if (!queries || !base || !scratch || !out_scores || !out_idx) return fail(ESMB200_EINVAL, "null argument");
  if (reinterpret_cast<uintptr_t>(queries) % 16 != 0 || reinterpret_cast<uintptr_t>(base) % 16 != 0)
    return fail(ESMB200_EINVAL, "knn_search needs 16-byte aligned queries and base (TMA)");
  if (reinterpret_cast<uintptr_t>(scratch) % 16 != 0) return fail(ESMB200_EINVAL, "scratch must be 16-byte aligned");
  if (scratch_bytes < (size_t)splits * (size_t)Q * (size_t)k * 8)
    return fail(ESMB200_EINVAL, "scratch smaller than esmb200_knn_scratch_bytes");
  if (Q == 0) return ESMB200_OK;
  int rc = check_device();
  if (rc) return rc;
  CUtensorMap tq, tx;
  if ((rc = make_tmap_f16(&tq, queries, (uint64_t)Q, (uint64_t)D, (uint64_t)q_ld, knn_cfg::BLOCK_M))) return rc;
  if ((rc = make_tmap_f16(&tx, base, (uint64_t)N, (uint64_t)D, (uint64_t)b_ld, knn_cfg::BLOCK_N))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  KnnParams p;
  p.Q = Q;
  p.D = D;
  p.k = k;
  p.N = N;
  const int64_t tiles = (N + knn_cfg::BLOCK_N - 1) / knn_cfg::BLOCK_N;
  p.tiles_per_stripe = (int)((tiles + splits - 1) / splits);
  p.query_blocks = (Q + knn_cfg::BLOCK_M - 1) / knn_cfg::BLOCK_M;
  p.beta = beta;
  p.alpha = alpha;
  p.self_offset = self_offset;
  p.row0 = 0;
  p.seed = nullptr;
  p.keys = static_cast<unsigned long long*>(scratch);
  if ((rc = knn_launch_topk<false>(tq, tx, p, splits, st))) return rc;
  {
    ProfScope ps(T_KNN, st);
    const int threads = splits >= 256 ? 256 : (splits + 31) / 32 * 32;
    knn_merge_kernel<4, false><<<(unsigned)Q, threads, 0, st>>>(p.keys, Q, k, splits, nullptr, out_scores, out_idx);
    CK(cudaGetLastError());
  }
  return ESMB200_OK;
}

int esmb200_knn_search_accumulate(const void* queries, int64_t q_ld, int32_t Q, const void* base, int64_t b_ld,
                                  int64_t n, int64_t row0, int32_t D, const float* beta, float alpha,
                                  int64_t self_offset, int32_t k, int32_t splits, void* scratch, size_t scratch_bytes,
                                  uint64_t* keys, void* stream) {
  if (k < 1 || k > knn_cfg::MAX_K) return fail(ESMB200_EINVAL, "knn_search_accumulate needs 1 <= k <= 128");
  if (Q < 0 || n < 1 || row0 < 0 || row0 > INT32_MAX || n > INT32_MAX - row0)
    return fail(ESMB200_EINVAL, "knn_search_accumulate needs Q >= 0, n >= 1, row0 >= 0 and row0 + n < 2^31");
  if (D < 64 || D % 64 != 0) return fail(ESMB200_EINVAL, "knn_search_accumulate needs D % 64 == 0");
  if (q_ld < D || b_ld < D || q_ld % 8 != 0 || b_ld % 8 != 0)
    return fail(ESMB200_EINVAL,
                "knn_search_accumulate needs q_ld, b_ld >= D and multiples of 8 (16-byte rows for TMA)");
  if (splits < 1 || splits > knn_cfg::MAX_SPLITS)
    return fail(ESMB200_EINVAL, "knn_search_accumulate needs 1 <= splits <= 1024");
  if (!queries || !base || !scratch || !keys) return fail(ESMB200_EINVAL, "null argument");
  if (reinterpret_cast<uintptr_t>(queries) % 16 != 0 || reinterpret_cast<uintptr_t>(base) % 16 != 0)
    return fail(ESMB200_EINVAL, "knn_search_accumulate needs 16-byte aligned queries and base (TMA)");
  if (reinterpret_cast<uintptr_t>(scratch) % 16 != 0) return fail(ESMB200_EINVAL, "scratch must be 16-byte aligned");
  if (reinterpret_cast<uintptr_t>(keys) % 8 != 0) return fail(ESMB200_EINVAL, "keys must be 8-byte aligned");
  if (scratch_bytes < (size_t)splits * (size_t)Q * (size_t)k * 8)
    return fail(ESMB200_EINVAL, "scratch smaller than esmb200_knn_scratch_bytes");
  if (Q == 0) return ESMB200_OK;
  int rc = check_device();
  if (rc) return rc;
  CUtensorMap tq, tx;
  if ((rc = make_tmap_f16(&tq, queries, (uint64_t)Q, (uint64_t)D, (uint64_t)q_ld, knn_cfg::BLOCK_M))) return rc;
  if ((rc = make_tmap_f16(&tx, base, (uint64_t)n, (uint64_t)D, (uint64_t)b_ld, knn_cfg::BLOCK_N))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  KnnParams p;
  p.Q = Q;
  p.D = D;
  p.k = k;
  p.N = n;
  const int64_t tiles = (n + knn_cfg::BLOCK_N - 1) / knn_cfg::BLOCK_N;
  p.tiles_per_stripe = (int)((tiles + splits - 1) / splits);
  p.query_blocks = (Q + knn_cfg::BLOCK_M - 1) / knn_cfg::BLOCK_M;
  p.beta = beta;
  p.alpha = alpha;
  p.self_offset = self_offset;
  p.row0 = row0;
  p.seed = reinterpret_cast<const unsigned long long*>(keys);
  p.keys = static_cast<unsigned long long*>(scratch);
  if ((rc = knn_launch_topk<true>(tq, tx, p, splits, st))) return rc;
  {
    ProfScope ps(T_KNN, st);
    const int lists = splits + 1;  // the stripes and the running list
    const int threads = lists >= 256 ? 256 : (lists + 31) / 32 * 32;
    knn_merge_kernel<5, true><<<(unsigned)Q, threads, 0, st>>>(p.keys, Q, k, splits,
                                                               reinterpret_cast<unsigned long long*>(keys), nullptr,
                                                               nullptr);
    CK(cudaGetLastError());
  }
  return ESMB200_OK;
}

int esmb200_knn_decode(const uint64_t* keys, int32_t Q, int32_t k, float* out_scores, int64_t* out_idx, void* stream) {
  if (Q < 0 || k < 1 || k > knn_cfg::MAX_K) return fail(ESMB200_EINVAL, "knn_decode needs Q >= 0 and 1 <= k <= 128");
  if (!keys || !out_scores || !out_idx) return fail(ESMB200_EINVAL, "null argument");
  if (reinterpret_cast<uintptr_t>(keys) % 8 != 0) return fail(ESMB200_EINVAL, "keys must be 8-byte aligned");
  if (reinterpret_cast<uintptr_t>(out_scores) % 4 != 0 || reinterpret_cast<uintptr_t>(out_idx) % 8 != 0)
    return fail(ESMB200_EINVAL, "knn_decode needs 4-byte aligned out_scores and 8-byte aligned out_idx");
  if (Q == 0) return ESMB200_OK;
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t total = (int64_t)Q * k;
  ProfScope ps(T_KNN, st);
  const int64_t blocks = (total + 255) / 256;
  knn_decode_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, st>>>(
      reinterpret_cast<const unsigned long long*>(keys), total, out_scores, out_idx);
  CK(cudaGetLastError());
  return ESMB200_OK;
}

int esmb200_knn_range(const void* queries, int64_t q_ld, int32_t Q, const void* base, int64_t b_ld, int64_t n,
                      int64_t row0, int32_t D, const float* beta, float alpha, int64_t self_offset, const float* tau,
                      int32_t splits, uint64_t* hit_keys, int32_t* hit_rows, int64_t hit_cap, uint64_t* hit_counts,
                      uint64_t* hit_total, void* stream) {
  if (Q < 0 || n < 1 || row0 < 0 || row0 > INT32_MAX || n > INT32_MAX - row0)
    return fail(ESMB200_EINVAL, "knn_range needs Q >= 0, n >= 1, row0 >= 0 and row0 + n < 2^31");
  if (D < 64 || D % 64 != 0) return fail(ESMB200_EINVAL, "knn_range needs D % 64 == 0");
  if (q_ld < D || b_ld < D || q_ld % 8 != 0 || b_ld % 8 != 0)
    return fail(ESMB200_EINVAL, "knn_range needs q_ld, b_ld >= D and multiples of 8 (16-byte rows for TMA)");
  if (splits < 1 || splits > knn_cfg::MAX_SPLITS) return fail(ESMB200_EINVAL, "knn_range needs 1 <= splits <= 1024");
  if (hit_cap < 0 || hit_cap > INT32_MAX) return fail(ESMB200_EINVAL, "knn_range needs 0 <= hit_cap < 2^31");
  if (!queries || !base || !tau || !hit_counts || !hit_total || (hit_cap > 0 && (!hit_keys || !hit_rows)))
    return fail(ESMB200_EINVAL, "null argument");
  if (reinterpret_cast<uintptr_t>(queries) % 16 != 0 || reinterpret_cast<uintptr_t>(base) % 16 != 0)
    return fail(ESMB200_EINVAL, "knn_range needs 16-byte aligned queries and base (TMA)");
  if (reinterpret_cast<uintptr_t>(beta) % 4 != 0 || reinterpret_cast<uintptr_t>(tau) % 4 != 0 ||
      reinterpret_cast<uintptr_t>(hit_rows) % 4 != 0 || reinterpret_cast<uintptr_t>(hit_keys) % 8 != 0 ||
      reinterpret_cast<uintptr_t>(hit_counts) % 8 != 0 || reinterpret_cast<uintptr_t>(hit_total) % 8 != 0)
    return fail(ESMB200_EINVAL, "knn_range needs 4-byte aligned beta, tau and hit_rows, 8-byte aligned hit_keys, "
                                "hit_counts and hit_total");
  if (Q == 0) return ESMB200_OK;
  int rc = check_device();
  if (rc) return rc;
  CUtensorMap tq, tx;
  if ((rc = make_tmap_f16(&tq, queries, (uint64_t)Q, (uint64_t)D, (uint64_t)q_ld, knn_cfg::BLOCK_M))) return rc;
  if ((rc = make_tmap_f16(&tx, base, (uint64_t)n, (uint64_t)D, (uint64_t)b_ld, knn_cfg::BLOCK_N))) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  KnnParams p = {};
  p.Q = Q;
  p.D = D;
  p.k = 1;
  p.N = n;
  const int64_t tiles = (n + knn_cfg::BLOCK_N - 1) / knn_cfg::BLOCK_N;
  p.tiles_per_stripe = (int)((tiles + splits - 1) / splits);
  p.query_blocks = (Q + knn_cfg::BLOCK_M - 1) / knn_cfg::BLOCK_M;
  p.beta = beta;
  p.alpha = alpha;
  p.self_offset = self_offset;
  p.row0 = row0;
  p.tau = tau;
  p.hit_keys = reinterpret_cast<unsigned long long*>(hit_keys);
  p.hit_rows = hit_rows;
  p.hit_counts = reinterpret_cast<unsigned long long*>(hit_counts);
  p.hit_total = reinterpret_cast<unsigned long long*>(hit_total);
  p.hit_cap = hit_cap;
  CK(cudaFuncSetAttribute(knn_topk_kernel<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                          knn_cfg::SMEM_BYTES));
  ProfScope ps(T_KNN, st);
  const int64_t grid = (int64_t)p.query_blocks * splits;
  knn_topk_kernel<false, false, true><<<(unsigned)grid, knn_cfg::NUM_THREADS, knn_cfg::SMEM_BYTES, st>>>(tq, tx, p);
  CK(cudaGetLastError());
  return ESMB200_OK;
}

int esmb200_knn_range_finish_scratch_bytes(int32_t Q, size_t* out) {
  if (!out) return fail(ESMB200_EINVAL, "null argument");
  if (Q < 0) return fail(ESMB200_EINVAL, "knn_range_finish_scratch_bytes needs Q >= 0");
  *out = ((size_t)Q + 1) * 8;
  return ESMB200_OK;
}

int esmb200_knn_range_finish(const uint64_t* keys, const int32_t* rows, int64_t nnz, const uint64_t* counts, int32_t Q,
                             int64_t max_hits, void* scratch, size_t scratch_bytes, int64_t* lims, float* scores,
                             int64_t* idx, void* stream) {
  if (Q < 0 || nnz < 0 || nnz > INT32_MAX)
    return fail(ESMB200_EINVAL, "knn_range_finish needs Q >= 0 and 0 <= nnz < 2^31");
  if (max_hits < 1 && max_hits != -1) return fail(ESMB200_EINVAL, "knn_range_finish needs max_hits >= 1, or -1");
  if (!counts || !scratch || !lims || (nnz > 0 && (!keys || !rows || !scores || !idx)))
    return fail(ESMB200_EINVAL, "null argument");
  if (reinterpret_cast<uintptr_t>(keys) % 8 != 0 || reinterpret_cast<uintptr_t>(rows) % 4 != 0 ||
      reinterpret_cast<uintptr_t>(counts) % 8 != 0 || reinterpret_cast<uintptr_t>(scratch) % 8 != 0 ||
      reinterpret_cast<uintptr_t>(lims) % 8 != 0 || reinterpret_cast<uintptr_t>(scores) % 4 != 0 ||
      reinterpret_cast<uintptr_t>(idx) % 8 != 0)
    return fail(ESMB200_EINVAL, "knn_range_finish needs 8-byte aligned keys, counts, scratch, lims and idx, 4-byte "
                                "aligned rows and scores");
  if (scratch_bytes < ((size_t)Q + 1) * 8)
    return fail(ESMB200_EINVAL, "scratch smaller than esmb200_knn_range_finish_scratch_bytes");
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  long long* off = static_cast<long long*>(scratch);
  {
    ProfScope ps(T_KNN, st);
    knn_range_scan_kernel<<<1, 1024, 0, st>>>(reinterpret_cast<const long long*>(counts), Q, max_hits, off,
                                              reinterpret_cast<long long*>(lims));
    CK(cudaGetLastError());
  }
  if (nnz == 0) return ESMB200_OK;
  ProfScope ps(T_KNN, st);
  const int64_t blocks = (nnz + 255) / 256;
  knn_range_decode_kernel<<<(unsigned)(blocks < 8192 ? blocks : 8192), 256, 0, st>>>(
      reinterpret_cast<const unsigned long long*>(keys), rows, nnz, Q, off, reinterpret_cast<const long long*>(lims),
      scores, idx);
  CK(cudaGetLastError());
  return ESMB200_OK;
}


extern "C++" {
namespace {
// Constants of the inverted-file search (esmb200_ivf_search); include/esmb200.h states them.
constexpr int kIvfExtraStripes = 64;  // probed lists: sum over the lists of their stripes beyond one is at most this
constexpr int kIvfAllCtas = 264;      // every list: stripes so that about two waves of a 132-SM H100 run
constexpr int kIvfMaxLists = 1 << 24;

// The scratch of one esmb200_ivf_search call: every region's byte offset, from the arguments alone.
struct IvfLayout {
  bool all;
  int T, R;          // tiles per stripe; partial lists per query (stride)
  int64_t P;         // gathered query rows (probed) or Q (all)
  int64_t max_items;
  size_t cnt, gstart, istart, slot, pbase, gq, gself, counts, items, qg, keys, bytes;
};

IvfLayout ivf_layout(int Q, int nprobe, int nlist, int64_t N, int D, int k) {
  IvfLayout L{};
  L.all = nprobe == nlist;
  const int64_t tiles = (N + knn_cfg::BLOCK_N - 1) / knn_cfg::BLOCK_N;
  const int64_t blocks = ((int64_t)Q + knn_cfg::BLOCK_M - 1) / knn_cfg::BLOCK_M;
  if (L.all) {
    int64_t S = blocks > 0 ? (kIvfAllCtas + blocks - 1) / blocks : 1;
    S = S < tiles ? S : tiles;
    L.T = (int)((tiles + S - 1) / S);
    L.R = (int)((tiles + L.T - 1) / L.T);  // the stripes of T tiles
    L.P = Q;
    L.max_items = blocks * L.R;
  } else {
    const int64_t total = tiles + nlist;  // at least the sum over the lists of their tiles
    L.T = (int)((total + kIvfExtraStripes - 1) / kIvfExtraStripes);
    L.R = nprobe + kIvfExtraStripes;
    L.P = (int64_t)Q * nprobe;
    L.max_items = L.P / knn_cfg::BLOCK_M + (nlist < L.P ? nlist : L.P) + blocks * kIvfExtraStripes;
  }
  size_t o = 0;
  auto take = [&](size_t bytes) {
    const size_t at = o;
    o += (bytes + 255) / 256 * 256;
    return at;
  };
  const size_t P = (size_t)L.P, nl = L.all ? 0 : (size_t)nlist + 1;
  L.cnt = take(nl * 4);
  L.gstart = take(nl * 4);
  L.istart = take(nl * 4);
  L.slot = take(L.all ? 0 : P * 4);
  L.pbase = take(P * 4);
  L.gq = take(L.all ? 0 : P * 4);
  L.gself = take(L.all ? 0 : P * 8);
  L.counts = take((size_t)Q * 4);
  L.items = take((size_t)L.max_items * sizeof(IvfItem));
  L.qg = take(L.all ? 0 : P * (size_t)D * 2);
  L.keys = take((size_t)Q * L.R * (size_t)k * 8);
  L.bytes = o < 256 ? 256 : o;
  return L;
}

// the refusals the scratch size and the search share
int ivf_check(int32_t Q, int32_t nprobe, int32_t nlist, int64_t N, int32_t D, int32_t k, const char* what) {
  const std::string w(what);
  if (k < 1 || k > knn_cfg::MAX_K) return fail(ESMB200_EINVAL, w + " needs 1 <= k <= 128");
  if (Q < 0 || N < 1 || N > INT32_MAX) return fail(ESMB200_EINVAL, w + " needs Q >= 0 and 1 <= N < 2^31");
  if (nlist < 1 || nlist > kIvfMaxLists || nlist > N) return fail(ESMB200_EINVAL, w + " needs 1 <= nlist <= min(N, 2^24)");
  if (nprobe != nlist && (nprobe < 1 || nprobe > knn_cfg::MAX_K))
    return fail(ESMB200_EINVAL, w + " needs 1 <= nprobe <= min(nlist, 128) or nprobe == nlist");
  if (nprobe > nlist) return fail(ESMB200_EINVAL, w + " needs 1 <= nprobe <= min(nlist, 128) or nprobe == nlist");
  if (D < 64 || D % 64 != 0) return fail(ESMB200_EINVAL, w + " needs D % 64 == 0");
  if (nprobe != nlist && (int64_t)Q * nprobe > INT32_MAX / 2)
    return fail(ESMB200_EINVAL, w + " needs Q * nprobe < 2^30");
  // partial lists are indexed in int32: q * R + s for every query q and s < R
  if ((int64_t)Q * ivf_layout(Q, nprobe, nlist, N, D, k).R > INT32_MAX)
    return fail(ESMB200_EINVAL, w + " needs Q * R < 2^31 partial lists (R = nprobe + 64, or the stripes of every list)");
  return ESMB200_OK;
}
}  // namespace
}  // extern "C++"

int esmb200_ivf_scratch_bytes(int32_t Q, int32_t nprobe, int32_t nlist, int64_t N, int32_t D, int32_t k, size_t* out) {
  if (!out) return fail(ESMB200_EINVAL, "null argument");
  int rc = ivf_check(Q, nprobe, nlist, N, D, k, "ivf_scratch_bytes");
  if (rc) return rc;
  *out = ivf_layout(Q, nprobe, nlist, N, D, k).bytes;
  return ESMB200_OK;
}

int esmb200_ivf_search(const void* queries, int64_t q_ld, int32_t Q, const void* rows, int64_t b_ld, int64_t N,
                       const int64_t* ids, const int64_t* offsets, int32_t nlist, int32_t D, const float* beta,
                       float alpha, const int32_t* probes, int32_t nprobe, const int64_t* self_ids, int32_t k,
                       void* scratch, size_t scratch_bytes, float* out_scores, int64_t* out_idx, void* stream) {
  int rc = ivf_check(Q, nprobe, nlist, N, D, k, "ivf_search");
  if (rc) return rc;
  const bool all = nprobe == nlist;
  if (q_ld < D || b_ld < D || q_ld % 8 != 0 || b_ld % 8 != 0)
    return fail(ESMB200_EINVAL, "ivf_search needs q_ld, b_ld >= D and multiples of 8 (16-byte rows for TMA)");
  if (!queries || !rows || !ids || !offsets || !scratch || !out_scores || !out_idx)
    return fail(ESMB200_EINVAL, "null argument");
  if (all != (probes == nullptr))
    return fail(ESMB200_EINVAL, "ivf_search needs probes NULL exactly when nprobe == nlist (every list)");
  if (reinterpret_cast<uintptr_t>(queries) % 16 != 0 || reinterpret_cast<uintptr_t>(rows) % 16 != 0)
    return fail(ESMB200_EINVAL, "ivf_search needs 16-byte aligned queries and rows (TMA)");
  if (reinterpret_cast<uintptr_t>(ids) % 8 != 0 || reinterpret_cast<uintptr_t>(offsets) % 8 != 0 ||
      reinterpret_cast<uintptr_t>(self_ids) % 8 != 0 || reinterpret_cast<uintptr_t>(probes) % 4 != 0 ||
      reinterpret_cast<uintptr_t>(beta) % 4 != 0)
    return fail(ESMB200_EINVAL, "ivf_search needs 8-byte aligned ids, offsets and self_ids, 4-byte aligned probes and beta");
  if (reinterpret_cast<uintptr_t>(out_scores) % 4 != 0 || reinterpret_cast<uintptr_t>(out_idx) % 8 != 0)
    return fail(ESMB200_EINVAL, "ivf_search needs 4-byte aligned out_scores and 8-byte aligned out_idx");
  if (reinterpret_cast<uintptr_t>(scratch) % 256 != 0) return fail(ESMB200_EINVAL, "scratch must be 256-byte aligned");
  const IvfLayout L = ivf_layout(Q, nprobe, nlist, N, D, k);
  if (scratch_bytes < L.bytes) return fail(ESMB200_EINVAL, "scratch smaller than esmb200_ivf_scratch_bytes");
  if (Q == 0) return ESMB200_OK;
  if ((rc = check_device())) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* sc = static_cast<uint8_t*>(scratch);
  int* cnt = reinterpret_cast<int*>(sc + L.cnt);
  int* gstart = reinterpret_cast<int*>(sc + L.gstart);
  int* istart = reinterpret_cast<int*>(sc + L.istart);
  int* slot = reinterpret_cast<int*>(sc + L.slot);
  int* pbase = reinterpret_cast<int*>(sc + L.pbase);
  int* gq = reinterpret_cast<int*>(sc + L.gq);
  int64_t* gself = reinterpret_cast<int64_t*>(sc + L.gself);
  int* counts = reinterpret_cast<int*>(sc + L.counts);
  IvfItem* items = reinterpret_cast<IvfItem*>(sc + L.items);
  __half* qg = reinterpret_cast<__half*>(sc + L.qg);
  int64_t n_items;
  const void* a_rows = queries;  // the query rows the list scan reads, and their leading dimension
  int64_t a_ld = q_ld;
  if (all) {
    n_items = ((int64_t)Q + knn_cfg::BLOCK_M - 1) / knn_cfg::BLOCK_M * L.R;
    ProfScope ps(T_KNN, st);
    const int64_t b = (n_items > Q ? n_items : Q) / 256 + 1;
    ivf_all_items_kernel<<<(unsigned)(b < 1024 ? b : 1024), 256, 0, st>>>(Q, N, L.R, L.T, items, pbase, counts);
    CK(cudaGetLastError());
  } else {
    CK(cudaMemsetAsync(cnt, 0, (size_t)nlist * 4, st));
    const int64_t P = L.P;
    {
      ProfScope ps(T_KNN, st);
      const int64_t b = (P + 255) / 256;
      ivf_count_kernel<<<(unsigned)(b < 4096 ? b : 4096), 256, 0, st>>>(probes, P, nprobe, nlist, cnt, slot);
      CK(cudaGetLastError());
    }
    {
      ProfScope ps(T_KNN, st);
      ivf_scan_kernel<<<1, 512, 0, st>>>(cnt, offsets, nlist, N, L.T, gstart, istart);
      CK(cudaGetLastError());
    }
    int host_items = 0;  // the one host synchronisation: the grid of the list scan
    CK(cudaMemcpyAsync(&host_items, istart + nlist, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    n_items = host_items;
    if (n_items > L.max_items) return fail(ESMB200_EINVAL, "ivf_search: offsets that do not partition [0, N)");
    {
      ProfScope ps(T_KNN, st);
      ivf_place_kernel<<<(unsigned)((Q + 255) / 256), 256, 0, st>>>(probes, slot, gstart, offsets, Q, nprobe, nlist, N,
                                                                    L.T, L.R, self_ids, gq, gself, pbase, counts);
      CK(cudaGetLastError());
    }
    {
      ProfScope ps(T_KNN, st);
      ivf_items_kernel<<<(unsigned)((nlist + 255) / 256), 256, 0, st>>>(cnt, gstart, istart, offsets, nlist, N, L.T,
                                                                        items);
      CK(cudaGetLastError());
    }
    {
      ProfScope ps(T_KNN, st);
      const int64_t b = (P * (D / 8) + 255) / 256;
      ivf_gather_kernel<<<(unsigned)(b < 8192 ? b : 8192), 256, 0, st>>>(static_cast<const __half*>(queries), q_ld,
                                                                         gq, gstart + nlist, D, qg);
      CK(cudaGetLastError());
    }
    a_rows = qg;
    a_ld = D;
  }
  if (n_items > 0) {
    CUtensorMap tq, tx;
    if ((rc = make_tmap_f16(&tq, a_rows, (uint64_t)L.P, (uint64_t)D, (uint64_t)a_ld, knn_cfg::BLOCK_M))) return rc;
    if ((rc = make_tmap_f16(&tx, rows, (uint64_t)N, (uint64_t)D, (uint64_t)b_ld, knn_cfg::BLOCK_N))) return rc;
    KnnParams p{};
    p.Q = (int)L.P;
    p.D = D;
    p.k = k;
    p.N = N;
    p.tiles_per_stripe = L.T;
    p.query_blocks = 1;
    p.beta = beta;
    p.alpha = alpha;
    p.self_offset = -1;
    p.row0 = 0;
    p.seed = nullptr;
    p.keys = reinterpret_cast<unsigned long long*>(sc + L.keys);
    p.items = items;
    p.ids = ids;
    p.gself = all ? self_ids : gself;
    p.pbase = pbase;
    CK(cudaFuncSetAttribute(knn_topk_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                            knn_cfg::SMEM_BYTES));
    ProfScope ps(T_KNN, st);
    knn_topk_kernel<false, true><<<(unsigned)n_items, knn_cfg::NUM_THREADS, knn_cfg::SMEM_BYTES, st>>>(tq, tx, p);
    CK(cudaGetLastError());
  }
  {
    ProfScope ps(T_KNN, st);
    knn_merge_kernel<2, false, true><<<(unsigned)Q, 256, 0, st>>>(
        reinterpret_cast<const unsigned long long*>(sc + L.keys), Q, k, L.R, nullptr, out_scores, out_idx, counts);
    CK(cudaGetLastError());
  }
  return ESMB200_OK;
}

int esmb200_kmeans_means(const void* rows, int64_t ld, int64_t n, int32_t D, const int64_t* assign, int32_t nlist,
                         int64_t* sums, float* means_out, int64_t* counts_out, void* stream) {
  if (n < 0 || n > (int64_t(1) << 23))
    return fail(ESMB200_EINVAL, "kmeans_means needs 0 <= n <= 2^23 (so no int64 column sum can overflow)");
  if (D < 8 || D % 8 != 0 || ld < D || ld % 8 != 0)
    return fail(ESMB200_EINVAL, "kmeans_means needs D % 8 == 0 and ld >= D, a multiple of 8");
  if (nlist < 1 || nlist > kIvfMaxLists) return fail(ESMB200_EINVAL, "kmeans_means needs 1 <= nlist <= 2^24");
  if (!rows || !assign || !sums || !means_out || !counts_out) return fail(ESMB200_EINVAL, "null argument");
  if (reinterpret_cast<uintptr_t>(rows) % 16 != 0 || reinterpret_cast<uintptr_t>(assign) % 8 != 0 ||
      reinterpret_cast<uintptr_t>(sums) % 8 != 0 || reinterpret_cast<uintptr_t>(counts_out) % 8 != 0 ||
      reinterpret_cast<uintptr_t>(means_out) % 4 != 0)
    return fail(ESMB200_EINVAL, "kmeans_means needs 16-byte aligned rows, 8-byte aligned assign, sums and counts");
  if ((int64_t)nlist * D > (int64_t(1) << 40)) return fail(ESMB200_EINVAL, "kmeans_means needs nlist * D <= 2^40");
  int rc = check_device();
  if (rc) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  CK(cudaMemsetAsync(sums, 0, (size_t)nlist * D * 8, st));
  CK(cudaMemsetAsync(counts_out, 0, (size_t)nlist * 8, st));
  if (n > 0) {
    ProfScope ps(T_KNN, st);
    const int64_t b = (n + 7) / 8;
    kmeans_sum_kernel<<<(unsigned)(b < 8192 ? b : 8192), 256, 0, st>>>(
        static_cast<const __half*>(rows), ld, n, D, assign, nlist, reinterpret_cast<unsigned long long*>(sums),
        reinterpret_cast<unsigned long long*>(counts_out));
    CK(cudaGetLastError());
  }
  {
    ProfScope ps(T_KNN, st);
    const int64_t b = ((int64_t)nlist * D + 255) / 256;
    kmeans_mean_kernel<<<(unsigned)(b < 8192 ? b : 8192), 256, 0, st>>>(
        reinterpret_cast<const long long*>(sums), reinterpret_cast<const long long*>(counts_out), nlist, D, means_out);
    CK(cudaGetLastError());
  }
  return ESMB200_OK;
}

size_t esmb200_align_scratch_bytes(int32_t P, int64_t n_q, int64_t n_t, int64_t n_cells) {
  if (P < 0 || n_q < 0 || n_t < 0 || n_cells < 0) return 0;
  return align_scratch(P, n_q, n_t, n_cells).bytes;
}

namespace {
// the refusals both alignment calls share; the per-pair offsets are the caller's (esm_b200/align.py builds them)
int align_check(const int64_t* q_off, const int64_t* t_off, const int64_t* s_off, int32_t P, int64_t n_q, int64_t n_t,
                int64_t n_cells, const void* scratch, size_t scratch_bytes) {
  if (P < 0) return fail(ESMB200_EINVAL, "align needs P >= 0");
  if (n_q < P || n_t < P || n_cells < P || n_q > INT32_MAX * (int64_t)P || n_t > INT32_MAX * (int64_t)P)
    return fail(ESMB200_EINVAL, "align needs La, Lb >= 1 for every pair: n_q, n_t and n_cells >= P");
  if (n_cells > (int64_t(1) << 40)) return fail(ESMB200_EINVAL, "align needs n_cells <= 2^40");
  if (P == 0) return ESMB200_OK;
  if (!q_off || !t_off || !s_off || !scratch) return fail(ESMB200_EINVAL, "null argument");
  if (reinterpret_cast<uintptr_t>(scratch) % 256 != 0) return fail(ESMB200_EINVAL, "scratch must be 256-byte aligned");
  if (scratch_bytes < align_scratch(P, n_q, n_t, n_cells).bytes)
    return fail(ESMB200_EINVAL, "more cells than the scratch: scratch smaller than esmb200_align_scratch_bytes");
  return ESMB200_OK;
}

unsigned align_splits(int32_t P, int per_sm) {  // CTAs per pair: fill the GPU about per_sm times over
  const int64_t want = ((int64_t)per_sm * num_sms() + P - 1) / P;
  return (unsigned)(want < 1 ? 1 : want > 64 ? 64 : want);
}
}  // namespace

int esmb200_align_similarity(const void* q_rows, const void* t_rows, int32_t D, const int64_t* q_off,
                             const int64_t* t_off, const int64_t* s_off, int32_t P, int64_t n_q, int64_t n_t,
                             int64_t n_cells, int32_t zscore, float* out, void* scratch, size_t scratch_bytes,
                             void* stream) {
  if (D < 64 || D % 64 != 0) return fail(ESMB200_EINVAL, "align_similarity needs D % 64 == 0");
  if (zscore != 0 && zscore != 1) return fail(ESMB200_EINVAL, "align_similarity zscore must be 0 or 1");
  int rc = align_check(q_off, t_off, s_off, P, n_q, n_t, n_cells, scratch, scratch_bytes);
  if (rc || P == 0) return rc;
  if (!q_rows || !t_rows || !out) return fail(ESMB200_EINVAL, "null argument");
  if (reinterpret_cast<uintptr_t>(q_rows) % 16 != 0 || reinterpret_cast<uintptr_t>(t_rows) % 16 != 0)
    return fail(ESMB200_EINVAL, "align_similarity needs 16-byte aligned rows");
  if ((rc = check_device())) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const AlignScratch sc = align_scratch(P, n_q, n_t, n_cells);
  float2* stats = reinterpret_cast<float2*>(static_cast<char*>(scratch) + sc.stats_off);
  {  // one ProfScope per kernel: esmb200_launch_count counts kernels
    ProfScope ps(T_ALIGN, st);
    align_sim_kernel<<<dim3((unsigned)P, align_splits(P, 8)), kAlignSimThreads, 0, st>>>(
        static_cast<const __half*>(q_rows), static_cast<const __half*>(t_rows), D, q_off, t_off, s_off, out);
    CK(cudaGetLastError());
  }
  if (zscore) {
    {
      ProfScope ps(T_ALIGN, st);
      align_stats_kernel<<<dim3((unsigned)P, align_splits(P, 8)), kAlignStatThreads, 0, st>>>(out, q_off, t_off, s_off,
                                                                                               n_q, stats);
      CK(cudaGetLastError());
    }
    ProfScope ps(T_ALIGN, st);
    align_zscore_kernel<<<dim3((unsigned)P, align_splits(P, 8)), kAlignStatThreads, 0, st>>>(out, q_off, t_off, s_off,
                                                                                              n_q, stats);
    CK(cudaGetLastError());
  }
  return ESMB200_OK;
}

int esmb200_align(const float* s, const int64_t* q_off, const int64_t* t_off, const int64_t* s_off, int32_t P,
                  int64_t n_q, int64_t n_t, int64_t n_cells, int32_t mode, float gap_open, float gap_extend,
                  void* scratch, size_t scratch_bytes, float* scores, int32_t* spans, uint8_t* ops, int32_t* n_ops,
                  void* stream) {
  if (mode != ESMB200_ALIGN_LOCAL && mode != ESMB200_ALIGN_GLOBAL)
    return fail(ESMB200_EINVAL, "align mode must be ESMB200_ALIGN_LOCAL or ESMB200_ALIGN_GLOBAL");
  if (!(gap_open >= 0.f) || !(gap_extend >= 0.f) || !isfinite(gap_open) || !isfinite(gap_extend))
    return fail(ESMB200_EINVAL, "align needs finite gap penalties >= 0");
  int rc = align_check(q_off, t_off, s_off, P, n_q, n_t, n_cells, scratch, scratch_bytes);
  if (rc || P == 0) return rc;
  if (!s || !scores || !spans || !ops || !n_ops) return fail(ESMB200_EINVAL, "null argument");
  if ((rc = check_device())) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const AlignScratch sc = align_scratch(P, n_q, n_t, n_cells);
  uint8_t* base = static_cast<uint8_t*>(scratch);
  const int local = mode == ESMB200_ALIGN_LOCAL;
  {
    ProfScope ps(T_ALIGN, st);
    align_dp_kernel<<<(unsigned)P, 32, 0, st>>>(s, q_off, t_off, s_off, local, gap_open, gap_extend, base,
                                                sc.border_off, scores, spans);
    CK(cudaGetLastError());
  }
  {
    ProfScope ps(T_ALIGN, st);
    align_trace_kernel<<<(unsigned)((P + 127) / 128), 128, 0, st>>>(q_off, t_off, s_off, P, local, base, spans, ops,
                                                                    n_ops);
    CK(cudaGetLastError());
  }
  return ESMB200_OK;
}


int esmb200_set_option(const char* name, int32_t value) {
  if (!name) return fail(ESMB200_EINVAL, "null option name");
  if (!strcmp(name, "pdl") && (value == 0 || value == 1)) { pdl_flag() = value; return ESMB200_OK; }
  return fail(ESMB200_EINVAL, std::string("unknown option or value: ") + name);
}

long long esmb200_launch_count(void) {
  std::lock_guard<std::mutex> lk(g_prof.mu);
  return g_prof.launches;
}

int esmb200_profile_enable(int32_t max_launches) {
  std::lock_guard<std::mutex> lk(g_prof.mu);
  for (cudaEvent_t e : g_prof.ev) cudaEventDestroy(e);
  g_prof.ev.clear();
  g_prof.tag.clear();
  g_prof.used = 0;
  g_prof.on = max_launches > 0;
  for (int i = 0; i < 2 * max_launches; ++i) {
    cudaEvent_t e;
    CK(cudaEventCreate(&e));
    g_prof.ev.push_back(e);
  }
  return ESMB200_OK;
}

int esmb200_profile_read(int32_t* tags, float* ms, int32_t max_records) {
  std::lock_guard<std::mutex> lk(g_prof.mu);
  const int n = (int)(g_prof.used / 2);
  int out = 0;
  for (int i = 0; i < n && out < max_records; ++i, ++out) {
    CK(cudaEventSynchronize(g_prof.ev[2 * i + 1]));
    float t = 0.f;
    CK(cudaEventElapsedTime(&t, g_prof.ev[2 * i], g_prof.ev[2 * i + 1]));
    tags[out] = g_prof.tag[i];
    ms[out] = t;
  }
  g_prof.used = 0;
  g_prof.tag.clear();
  return out;
}

}  // extern "C"
