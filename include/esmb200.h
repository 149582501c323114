/* esmb200.h — C ABI of the H100-native ESM-2 transformer-layer forward path (libesmb200.so).
 *
 * The reference (facebookresearch/esm, fair-esm 2.0.1) is pure Python and has no FFI for this path; the seam this
 * library sits behind is the Python method
 *     esm.modules.TransformerLayer.forward(x, self_attn_mask, self_attn_padding_mask, need_head_weights)
 *                                                      /root/reference/esm/modules.py:120-142
 * called from ESM2.forward's layer loop                 /root/reference/esm/model/esm2.py:111-121
 * Each entry point below names the reference code it replaces. The reference-side binding (a ctypes stub) is shown in
 * INTEGRATION.md; esm_b200/_lib.py is the shipped copy of that binding.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer owned by the caller (PyTorch), borrowed for the duration of the call;
 *     the library owns only its packed fp16 weight copies inside esmb200_layer
 *   - calls are asynchronous on `stream` (a cudaStream_t passed as void*), never synchronise
 *   - return 0 on success, a negative ESMB200_E* code on failure; esmb200_last_error() gives the message of the last
 *     failure on the calling thread. A device out-of-memory message starts with "CUDA out of memory" so that
 *     scripts/fold.py:165-178's handler keeps working
 *   - activations: residual stream x is fp32 [B, T, E] row-major (batch-major, i.e. the reference's (T,B,E)
 *     transposed); MMA operands are fp16 with fp32 accumulation; LayerNorm / softmax / residual adds are fp32
 *   - even head_dim <= 128 (every esm.pretrained.esm2_* model; heads narrower than 64 run in zero-padded 64-wide
 *     slots, 128-wide heads in two); no CPU fallback
 *   - ESM-1b / ESM-1v (esm/model/esm1.py, arch roberta_large) run the same layers without rotary tables, after
 *     esmb200_esm1b_embed
 *   - variant-effect scoring (examples/variant-prediction/predict.py; esm_b200.variants) batches the masked copies
 *     into one esmb200_stack_forward per chunk, runs the LM head on the masked rows only and finishes with
 *     esmb200_log_softmax_rows
 */
#ifndef ESMB200_H_
#define ESMB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ESMB200_OK 0
#define ESMB200_EINVAL -1   /* bad argument / unsupported shape */
#define ESMB200_ECUDA -2    /* CUDA runtime or driver error */
#define ESMB200_ENOMEM -3   /* device allocation failed ("CUDA out of memory ...") */
#define ESMB200_EWORKSPACE -4 /* workspace too small */

#define ESMB200_ABI_VERSION 4

typedef struct esmb200_layer esmb200_layer; /* opaque: packed weights + TMA descriptors of one TransformerLayer */

/* fp32 device pointers to one layer's parameters, nn.Linear layout weight[out,in] (state-dict names in comments,
 * prefix "layers.{i}."; /root/reference/esm/modules.py:99-118, multihead_attention.py:109-113) */
typedef struct esmb200_layer_weights {
  int32_t embed_dim;   /* E */
  int32_t num_heads;   /* H, E == head_dim * H */
  int32_t ffn_dim;     /* F = 4E */
  float ln_eps;        /* 1e-5 */
  const float* ln1_weight; /* self_attn_layer_norm.weight [E] */
  const float* ln1_bias;   /* self_attn_layer_norm.bias   [E] */
  const float* q_weight;   /* self_attn.q_proj.weight [E,E] */
  const float* q_bias;     /* self_attn.q_proj.bias   [E]   */
  const float* k_weight;   /* self_attn.k_proj.weight [E,E] */
  const float* k_bias;
  const float* v_weight;   /* self_attn.v_proj.weight [E,E] */
  const float* v_bias;
  const float* out_weight; /* self_attn.out_proj.weight [E,E] */
  const float* out_bias;
  const float* ln2_weight; /* final_layer_norm.weight [E] */
  const float* ln2_bias;
  const float* fc1_weight; /* fc1.weight [F,E]; NULL = attention-only layer (no ln2/fc1/fc2; esmb200_axial_stack_forward) */
  const float* fc1_bias;   /* fc1.bias   [F]   */
  const float* fc2_weight; /* fc2.weight [E,F] */
  const float* fc2_bias;   /* fc2.bias   [E]   */
  int32_t head_dim;        /* 0 = E / H. Even values <= 128. 16 / 24 / 32 (ESM-2 8M / 35M / 150M) run in zero-padded
                            * 64-wide head slots of the attention-side tensors; 64 = 650M / 3B / MSA Transformer;
                            * 65..128 (15B: 128) take two slots per head and 64-column rope tables */
  int32_t precision;       /* 0 = fp16 MMA operands (default). 1 = "fp32x3": every MMA operand (activations, weights,
                            * q, k, v, P) is an fp16 hi | lo pair and every product runs hi*hi + lo*hi + hi*lo into the
                            * fp32 accumulator (22 significand bits per operand) — fp32-grade results at ~3x the tensor
                            * work; needs E % 64 == 0 and head_dim <= 64. On the MSA axial path every row and
                            * column layer of one esmb200_axial_stack_forward call must share the precision.
                            * 2 = "fp8": the QKV, fc1 and fc2 projections run e4m3 x e4m3 wgmma GEMMs with power-of-two
                            * block scales (activations one per row and 128 columns, weights one per 128 x 128 block)
                            * and an fp32 promotion per 128-wide K block; LayerNorm writes e4m3 + scales, fc1's
                            * epilogue writes fc2's e4m3 operand + scales. Attention, out_proj, the residual stream
                            * and the contact pass are those of precision 0. Needs a feed-forward layer with
                            * ffn_dim % 128 == 0; not for the MSA axial stack (ESMB200_EINVAL) and not offloadable
                            * (esmb200_layer_packed_bytes is 0, esmb200_layer_offload ESMB200_EINVAL) */
} esmb200_layer_weights;

int esmb200_abi_version(void);
const char* esmb200_last_error(void);

/* Packs one TransformerLayer's weights (fp32 -> fp16, [Wq;Wk;Wv] concatenated) on `stream`.
 * Replaces TransformerLayer.__init__/_init_submodules state, modules.py:87-118. */
int esmb200_layer_create(const esmb200_layer_weights* w, void* stream, esmb200_layer** out);
int esmb200_layer_destroy(esmb200_layer* layer);

/* Scratch bytes needed by esmb200_layer_forward / esmb200_stack_forward for a [B,T] batch. */
size_t esmb200_workspace_bytes(int32_t embed_dim, int32_t num_heads, int32_t ffn_dim, int32_t B, int32_t T,
                               int32_t precision);

/* One TransformerLayer.forward (modules.py:120-142), in place on x:
 *     x += out_proj(attention(rope(q_proj(LN1 x) * d^-1/2), rope(k_proj(LN1 x)), v_proj(LN1 x)));
 *     x += fc2(gelu(fc1(LN2 x)))
 *   x          fp32 [B,T,E], updated in place
 *   pad_mask   uint8/bool [B,T], nonzero = padding key (self_attn_padding_mask, esm2.py:82), or NULL
 *   rope_cos/sin fp32 [T,32] (head_dim <= 64) or [T,64] (head_dim <= 128): cos/sin(t * inv_freq[j]) for j < head_dim/2
 *              (rotary_embedding.py:47-61), built by the caller; columns >= head_dim/2 are ignored.
 *              Both NULL: no rotary embedding, q and k stay unrotated (ESM-1b / ESM-1v layers, whose positions are
 *              added by esmb200_esm1b_embed; multihead_attention.py:354 with rot_emb = None). Exactly one NULL is
 *              ESMB200_EINVAL. The same holds for esmb200_stack_forward.
 *   attn_probs fp32 [B,H,T,T] or NULL: softmax probabilities per head (need_head_weights=True,
 *              multihead_attention.py:397-400, batch-major i.e. already transposed as esm2.py:121 does) */
int esmb200_layer_forward(esmb200_layer* layer, float* x, const uint8_t* pad_mask, int32_t B, int32_t T,
                          const float* rope_cos, const float* rope_sin, float* attn_probs, void* workspace,
                          size_t workspace_bytes, void* stream);

/* Optional contact-head accumulation fused into the need_head_weights pass of esmb200_stack_forward
 * (ContactPredictionHead.forward esm/modules.py:338-357, restated as in esmb200_contact_accumulate): every layer's
 * probabilities are folded into the accumulators while they are written, the stacked attention tensor is never read
 * back. S = hi - lo, nt = ceil(T / 128). Ignored (the separate probability kernel runs) for fp32x3 layers. */
typedef struct esmb200_contact_job {
  const float* weights; /* [n_layers, H] fp32: contact_head.regression.weight */
  const uint8_t* keep;  /* [B,T] 1 = not <eos>, or NULL */
  float* acc;           /* [B,S,S]  += sum_{l,h} w[l,h] A_{l,h}; zeroed by the caller */
  float* row_part;      /* [n_layers,B,H,4*nt,S] row sums of A_{l,h} per 32-key quarter tile (sum over 4*nt = rowsum) */
  float* col_part;      /* [n_layers,B,H,4*nt,S] column sums per 32-query quarter tile (sum over 4*nt = colsum) */
  int32_t lo, hi;       /* cropped positions [lo,hi): 1 .. T-1 for <cls> ... <eos> */
} esmb200_contact_job;

/* The layer loop of ESM2.forward (esm2.py:111-121), and of ProteinBertModel.forward for ESM-1b / ESM-1v (esm1.py:155-163)
 * with rope_cos == rope_sin == NULL: runs n_layers layers in place on x.
 *   repr_out[i]  NULL or fp32 [B,T,E]: copy of x after layer i (hidden_representations[i+1], esm2.py:117-118)
 *   attn_out[i]  NULL or fp32 [B,H,T,T]: attention probabilities of layer i (esm2.py:119-121); batch b starts at
 *                attn_out[i] + b * attn_batch_stride elements (0 = contiguous H*T*T), so the caller can point layer i
 *                into its slice of the stacked [B,L,H,T,T] result (esm2.py:134) and skip the torch.stack copy;
 *                attn_flags bit 0: write the rows of padded QUERY tokens as zeros (esm2.py:135-139; padded key
 *                columns are zero anyway), so the caller needs no masking pass over the stack
 * either array pointer itself may be NULL. */
int esmb200_stack_forward(esmb200_layer* const* layers, int32_t n_layers, float* x, const uint8_t* pad_mask,
                          int32_t B, int32_t T, const float* rope_cos, const float* rope_sin,
                          float* const* repr_out, float* const* attn_out, int64_t attn_batch_stride,
                          int32_t attn_flags, const esmb200_contact_job* contact /* nullable */, void* workspace,
                          size_t workspace_bytes, void* stream);

/* ---- streamed weights: a stack whose packed matrices live in pinned host memory (ESM-2 15B on one GPU; the
 * reference's CPU offloading, examples/esm2_infer_fairscale_fsdp_cpu_offloading.py, scripts/fold.py --cpu-offload) ----
 * esmb200_layer_packed_bytes: bytes of one layer's packed matrices (w_qkv, w_out, w_fc1, w_fc2, each 1024-aligned,
 *   back to back): the size of its host copy and of one ring slot. Pure host arithmetic; 0 for an unsupported shape.
 * esmb200_layer_offload: copies the packed matrices into host_dst (pinned, caller-owned, at least
 *   esmb200_layer_packed_bytes; it must outlive the layer) after the work queued on `stream` (esmb200_layer_create's
 *   packing), synchronises `stream`, and frees their device copies. The packed q/k/v bias and the borrowed LayerNorm
 *   vectors and biases stay on the device. From then on esmb200_layer_forward and esmb200_stack_forward return
 *   ESMB200_EINVAL for the layer and launch nothing; esmb200_stack_forward_streamed runs it.
 * esmb200_stack_forward_streamed: esmb200_stack_forward (same arguments and results, bit-identical) on layers that are
 *   all offloaded and share E, H, F and precision; a handle may appear more than once. ring: a device buffer of at
 *   least 2 * esmb200_layer_packed_bytes (16-byte aligned). Layer i's matrices are copied into slot i % 2 on
 *   copy_stream (a stream other than `stream`, so that the copies run on the copy engine under the previous layer's
 *   kernels), once layer i - 2's fc2 GEMM has run; layer i's QKV GEMM waits for its copy. copy_stream first waits
 *   for the work already queued on `stream`, and `stream` waits for every copy of the call, so calls that share a
 *   ring on one stream, and the caller's stream-ordered reuse of the ring, are safe. */
size_t esmb200_layer_packed_bytes(int32_t embed_dim, int32_t num_heads, int32_t ffn_dim, int32_t precision);
int esmb200_layer_offload(esmb200_layer* layer, void* host_dst, size_t bytes, void* stream);
int esmb200_stack_forward_streamed(esmb200_layer* const* layers, int32_t n_layers, float* x, const uint8_t* pad_mask,
                                   int32_t B, int32_t T, const float* rope_cos, const float* rope_sin,
                                   float* const* repr_out, float* const* attn_out, int64_t attn_batch_stride,
                                   int32_t attn_flags, const esmb200_contact_job* contact /* nullable */,
                                   void* workspace, size_t workspace_bytes, void* ring, size_t ring_bytes,
                                   void* copy_stream, void* stream);

/* ---- contacts without the attention stack (ProteinLanguageModel.predict_contacts) ----
 * esmb200_stack_contacts: the layer loop of esmb200_stack_forward with a contact job and no attn_out. x, repr_out and
 *   the contacts are bit-identical to those of esmb200_stack_forward with attn_out for every layer, attn_flags = 1
 *   (padded query rows zero, as ESM2.forward asks) and the same job; the [B,L,H,T,T] stack is neither written nor
 *   needed. contact: required (NULL is ESMB200_EINVAL); acc zeroed by the caller. ring == NULL: every layer resident;
 *   otherwise every layer offloaded, with the ring, copy_stream and event protocol of esmb200_stack_forward_streamed.
 *   Mixed precision, or resident and offloaded layers mixed, is ESMB200_EINVAL.
 *   fp16 and fp8 layers: the fused pass without its probability stores (attention_contact.cuh); row_part and col_part
 *     have the esmb200_contact_job layout [n_layers,B,H,4*nt,S]. probs_scratch is not used and may be NULL.
 *   fp32x3 layers: per layer, the split probability kernel writes the maps into probs_scratch (fp32 [B,H,T,T], 16-byte
 *     aligned), then esmb200_contact_accumulate's kernel reads them: row_part is row_sum [n_layers,B,H,S] and col_part
 *     is col_part [n_layers,B,H,ceil(S/16),S] of that entry, layer l at offset l*B*H*S and l*B*H*ceil(S/16)*S.
 *     a1 of layer l = row_part[l] + col_part[l] summed over its stripe axis. S <= 1024.
 *   A probs_scratch or workspace smaller than its size is ESMB200_EWORKSPACE. Every refusal comes before any launch.
 * esmb200_stack_contacts_bytes: bytes of row_part, col_part and probs_scratch for n_layers layers of num_heads heads,
 *   a [B,T] batch and S = hi - lo cropped positions in `precision` (0 fp16, 1 fp32x3, 2 fp8); scratch is 0 for 0 and 2.
 *   Pure host arithmetic; ESMB200_EINVAL for a non-positive size, S > T or an unknown precision. Out pointers may be
 *   NULL. */
int esmb200_stack_contacts_bytes(int32_t n_layers, int32_t num_heads, int32_t B, int32_t T, int32_t S,
                                 int32_t precision, size_t* row_part_bytes, size_t* col_part_bytes,
                                 size_t* scratch_bytes);
int esmb200_stack_contacts(esmb200_layer* const* layers, int32_t n_layers, float* x, const uint8_t* pad_mask, int32_t B,
                           int32_t T, const float* rope_cos, const float* rope_sin, float* const* repr_out,
                           const esmb200_contact_job* contact, void* probs_scratch, size_t probs_scratch_bytes,
                           void* workspace, size_t workspace_bytes, void* ring, size_t ring_bytes, void* copy_stream,
                           void* stream);

/* Embedding prologue of ESM2.forward (esm2.py:84-95): gather from table [V,E], zero <mask> rows and rescale by
 * 0.88/(1 - n_mask/n_nonpad) when token_dropout, zero pad rows. tokens int64 [B,T] -> x fp32 [B,T,E].
 * E % 4 == 0, B <= 65535. Pad rows are written as zeros whatever the scale: a sequence of pads only (scale 0/0) gives
 * zeros where the reference's x * (1 - padding_mask) keeps NaN. A sequence whose non-pad tokens are all <mask> (scale
 * 0.88/0) gives NaN at its non-pad rows, as the reference does. */
int esmb200_embed_tokens(const int64_t* tokens, const float* table, float* x, int32_t B, int32_t T, int32_t E,
                         int32_t padding_idx, int32_t mask_idx, int32_t token_dropout, void* stream);

/* Embedding prologue of ProteinBertModel.forward for ESM-1b / ESM-1v (esm/model/esm1.py:121-139), one launch:
 *   x = embed_table[tok]; token_dropout != 0: <mask> rows zeroed, x = (x * 0.88) / (1 - n_mask/n_nonpad);
 *   x += pos_table[cumsum(tok != pad) * (tok != pad) + padding_idx] (LearnedPositionalEmbedding, modules.py:240-257;
 *   a pad anywhere in the sequence is handled); ln_weight/ln_bias given: LayerNorm with eps (emb_layer_norm_before);
 *   pad rows zeroed.
 * tokens int64 [B,T]; embed_table [V,E]; pos_table [max_positions + padding_idx + 1, E] with T <= max_positions (the
 * caller checks, as the reference raises ValueError); ln_weight, ln_bias [E] both or neither. x fp32 [B,T,E].
 * E % 4 == 0, E <= 2560, T <= 12288. */
int esmb200_esm1b_embed(const int64_t* tokens, const float* embed_table, const float* pos_table, const float* ln_weight,
                        const float* ln_bias, float eps, int32_t token_dropout, int32_t padding_idx, int32_t mask_idx,
                        float* x, int32_t B, int32_t T, int32_t E, void* stream);

/* torch.nn.LayerNorm over the last dim (ESM1bLayerNorm, modules.py:68-81; emb_layer_norm_after, esm2.py:123):
 * fp32 [M,E] -> fp32 [M,E]. out may alias x. */
int esmb200_layernorm(const float* x, const float* weight, const float* bias, float* out, int32_t M, int32_t E,
                      float eps, void* stream);

/* Per-sequence mean representation, scripts/extract.py:116-119: out[b] = mean_t x[b, 1 : 1+lengths[b]] (residues only,
 * <cls> at position 0 excluded). x fp32 [B,T,E], lengths int32 [B] (device), out fp32 [B,E]. T >= 2, E % 4 == 0.
 * lengths[b] is clamped to [0, T-1] as the slice clamps it; 0 gives NaN (the mean of an empty slice). Rows past the
 * length and the <cls> row are not read. Deterministic. */
int esmb200_mean_pool(const float* x, const int32_t* lengths, float* out, int32_t B, int32_t T, int32_t E,
                      void* stream);

/* log_softmax over the first V columns of each row (examples/variant-prediction/predict.py:142,175,194,211:
 * torch.log_softmax(logits, -1)), fp32, one warp per row: row max, sum of expf(x - max), logf (accurate, not
 * ex2.approx: matches torch.log_softmax to ~1e-6). logits fp32 [n, ld], V <= ld, V <= 64.
 * target NULL: out fp32 [n, V]. target int64 [n]: out fp32 [n] = the log-probability of column target[i]
 * (predict.py:114,143). Targets must lie in [0, V); the caller checks them. n == 0 launches nothing. */
int esmb200_log_softmax_rows(const float* logits, int64_t ld, int32_t n, int32_t V, const int64_t* target,
                             float* out, void* stream);

/* Overlapping-window merge (esm_b200/windows.py: a protein longer than the window runs as overlapping crops whose
 * rows are stitched back together): a segmented weighted row sum
 *     out[r, c] = sum over j in [seg[r], seg[r+1]) of w[j] * src[idx[j], c],   r < rows, c < C,
 * the terms taken in j order as one fp32 fma chain per element. A segment of one term is copied bit for bit (weight
 * ignored; -0.0 and NaN pass through), an empty segment writes +0. src fp32 [*, src_ld], out fp32 [rows, out_ld]
 * (must not overlap src); idx int64, w fp32 and seg int64 [rows + 1] are device arrays, seg non-decreasing and every
 * idx[j] a valid src row (the caller builds them). Any C (33 logits, E-wide representations). Deterministic, no
 * atomics. rows == 0 launches nothing. */
int esmb200_window_merge(const float* src, int64_t src_ld, const int64_t* idx, const float* w, const int64_t* seg,
                         int32_t rows, int32_t C, float* out, int64_t out_ld, void* stream);

/* Categorical Jacobian contact map (esm_b200/jacobian.py; Zhang, Wayment-Steele, Brixi, Wang, Kern & Ovchinnikov,
 * PNAS 2024). A new operation with no reference code; its definition, for one protein of L residues:
 *   jac [L,20,L,20] fp32: J[i,a,j,b] = how the logit of amino acid b at residue j moves when residue i is set to amino
 *     acid a (20 amino acids "LAGVSERTIDPKQNFYMHWC"). Read only, never modified.
 *   Jc = J centred along each of its four axes (minus the mean over that axis; the four projections commute);
 *   N[i,j] = sqrt(sum_{a,b} Jc[i,a,j,b]^2), N[i,i] = 0;
 *   A = N - N.sum(1, keepdim) * N.sum(0, keepdim) / N.sum() (APC, as esm/modules.py:32-41), A[i,i] = 0;
 *   contacts [L,L] fp32 = (A + A^T) / 2. An all-zero J gives NaN off the diagonal (0 / 0), as the definition does.
 * Two passes over J (its marginal sums, then one 20 x 20 block norm per (i,j)) and a small L x L pass; every sum is
 * taken in fp64 in a fixed order, without atomics: the result is bit-reproducible. scratch:
 * esmb200_jacobian_scratch_bytes(L) bytes, 256-byte aligned (fp64 marginals and N, about 58 L^2 + 6,400 L bytes:
 * about 1/25 of J). 2 <= L <= 65535, else ESMB200_EINVAL, as is too little scratch; scratch_bytes(L < 2) is 0. */
size_t esmb200_jacobian_scratch_bytes(int32_t L);
int esmb200_jacobian_contacts(const float* jac, int32_t L, void* scratch, size_t scratch_bytes, float* contacts,
                              void* stream);

/* Gibbs sampling of protein sequences and MSA Transformer alignments (esm_b200/sampling.py). A new operation with no
 * reference code. Random stream: R(c0, c1, c2, c3) = Philox4x32-10 (curand_Philox4x32_10) with counter
 * (c0, c1, c2, c3) and key (seed mod 2^32, seed >> 32): four uint32 words. A word r maps to
 * u = ((r >> 8) + 0.5) * 2^-24 rounded toward zero to fp32, which lies in (0, 1) and is exact for u < 1/2. Every draw
 * depends only on (seed, chain, step, entry), never on how the chains are batched.
 * Layout: a chain is an alignment of R rows and C columns, column 0 <cls>, row-major; its residue entries (r, j),
 * 1 <= j < C, have the flat index p = r * W + (j - 1), W = C - 1, and p < 2^20. A protein of T tokens is R = 1,
 * C = T - 1: residue p is token 1 + p, and the <eos> column is never an entry.
 * esmb200_sample_order: the visiting order of one sweep. keys int64 [n_chains, n]:
 *     keys[c, j] = R(sweep, chain0 + c, p, 0).x * 2^20 + p,   p = entries[j],
 *   for the n designable entries entries int64 [n] (device; distinct, each in [0, 2^20), checked by the caller).
 *   Sorting each row ascending (keys are distinct) and taking key mod 2^20 gives the order; the caller sorts.
 *   n > 0, chain0 + n_chains <= 2^32, 0 <= sweep < 2^32, else ESMB200_EINVAL. n_chains == 0 launches nothing.
 * esmb200_sample_rows: one block update of step `step` for n / per_chain chains over the drawable token ids
 *   token_set int32 [n_tokens] (device, 1 <= n_tokens <= 32, each in [0, ld), checked by the caller), one warp per row,
 *   any n. Row r belongs to chain chain0 + r / per_chain (local chain r / per_chain) and resamples entry
 *   p = entries[r] (int64 [n], device). logits fp32 [n, ld]: the LM-head row of that entry of the chain's masked
 *   copy. For a < n_tokens:
 *     z_a = logits[r, token_set[a]] / temperature (fp32 division),
 *     g_a = -logf(-logf(u_a)), u_a from word a mod 4 of R(step, chain, p, 1 + a div 4),
 *     a* = argmax_a (z_a + g_a), a tie to the smallest a;
 *   tokens int64 (the chains' state, chain c at tokens + c * chain_stride) gets token_set[a*] at
 *   [c * chain_stride + (p / W) * C + 1 + p % W], in place; logq fp32 [n] gets (z_a* - max z) - logf(sum_a expf(z_a -
 *   max z)), bit for bit esmb200_log_softmax_rows' value with target a* on the n_tokens columns z. An entry outside
 *   [0, R * W) writes no token and a NaN logq. logp: NULL, or fp32 with logp[c * logp_stride] = the per_chain logq of
 *   local chain c summed in row order (fp32, from +0). ld >= 1, finite temperature > 0, R >= 1, C >= 2,
 *   chain_stride >= R * C, per_chain > 0 dividing n, chain0 + n / per_chain <= 2^32 and 0 <= step < 2^32, else
 *   ESMB200_EINVAL, before any launch. n == 0 launches nothing. Deterministic, no atomics. */
int esmb200_sample_order(const int64_t* entries, int32_t n, int32_t n_chains, int64_t chain0, int64_t sweep,
                         uint64_t seed, int64_t* keys, void* stream);
int esmb200_sample_rows(const float* logits, int64_t ld, int32_t n, const int32_t* token_set, int32_t n_tokens,
                        float temperature, uint64_t seed, int64_t step, int64_t chain0, int32_t per_chain,
                        const int64_t* entries, int64_t* tokens, int64_t chain_stride, int32_t R, int32_t C,
                        float* logq, float* logp, int64_t logp_stride, void* stream);

/* Greedy row selection of a deep alignment for the MSA Transformer (esm_b200/msa_select.py): greedy_select of the
 * reference's examples/contact_prediction.ipynb ("MSA Transformer" section), which picks the rows fed to
 * predict_contacts, with the same rows for every input. rows uint8 [N, ld] (device, 16-byte aligned; ld % 16 == 0,
 * ld >= C, and the bytes in columns [C, ld) equal in every row, so they never differ); bytes are compared as bytes.
 * selected int64 [k] (device) receives the picked row indices in selection order:
 *   selected[0] = 0 (the query); for t = 1 ... k - 1:
 *     d_t[j]   = fp64(count_j / C), count_j = the columns in which row j differs from row selected[t - 1]
 *                (scipy's cdist(..., "hamming"));
 *     score[j] = pairwise_sum(d_1[j], ..., d_t[j]) / t in fp64, pairwise_sum numpy's: below 8 terms a sequential sum
 *                from +0; up to 128 eight strided accumulators r[i % 8] over the first n - n % 8 terms, combined as
 *                ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the tail added in order; above 128 the sums
 *                of the halves split at n / 2 - (n / 2) % 8 (the notebook's np.delete(..., axis=1).mean(0) reduces
 *                an F-contiguous array along its contiguous axis);
 *     selected[t] = the argmax (ESMB200_SELECT_MAX) or argmin (ESMB200_SELECT_MIN) of score over the rows not yet
 *                picked, a tie to the smallest index.
 *   The caller returns the rows unchanged when N <= k, and sorts the indices for the notebook's order.
 * One init launch and one launch per step; the picked index stays on the device, nothing synchronises with the host.
 * Deterministic. scratch: esmb200_msa_select_scratch_bytes(N, C, k) bytes, 256-byte aligned (uint16 counts
 * [k - 1, N] and O(N + C) more). 1 <= C <= 65535, 0 <= k <= N, a known mode, ld as above and enough scratch, else
 * ESMB200_EINVAL before any launch. k == 0 launches nothing. scratch_bytes of a negative argument is 0. */
#define ESMB200_SELECT_MAX 0
#define ESMB200_SELECT_MIN 1
size_t esmb200_msa_select_scratch_bytes(int32_t N, int32_t C, int32_t k);
int esmb200_msa_greedy_select(const uint8_t* rows, int64_t ld, int32_t N, int32_t C, int32_t k, int32_t mode,
                              int64_t* selected, void* scratch, size_t scratch_bytes, void* stream);

/* Exact k-nearest-neighbour search over embeddings (esm_b200/search.py). queries fp16 [Q, q_ld] and base fp16 [N, b_ld]
 * (device, 16-byte aligned, row-major, the first D columns used). For each query row i, the k largest of
 *     s(i, j) = alpha * (queries_i . base_j) + beta[j]      (fp32 accumulation of the fp16 products; beta NULL = 0)
 * over j in [0, N), leaving out j == i + self_offset when self_offset >= 0 (an all-against-all search passes 0),
 * ordered by (score descending, index ascending): out_scores fp32 [Q, k] and out_idx int64 [Q, k] (device, dense).
 * Cosine similarity: alpha 1, no beta, rows normalised before rounding to fp16. Squared Euclidean distance:
 * alpha 2, beta[j] = -|base_j|^2, so ranking by s descending ranks by distance ascending.
 * A query's results are bit-identical whatever the other queries, Q, its row or `splits`: a score depends only on its
 * two rows, and the top k under a total order does not depend on the order candidates are seen in.
 * Two launches: the fused wgmma GEMM + top-k over `splits` contiguous stripes of the database, one partial top k per
 * (query, stripe) into scratch, then a merge of the stripes' lists per query. The score matrix is never stored.
 * scratch: esmb200_knn_scratch_bytes(Q, k, splits) bytes, 16-byte aligned. 1 <= k <= 128, k <= N (k <= N - 1 with
 * self_offset >= 0), 1 <= N < 2^31, Q >= 0, D % 64 == 0, q_ld and b_ld >= D and multiples of 8, 1 <= splits <= 1024,
 * non-NULL pointers and enough scratch, else ESMB200_EINVAL before any launch. Q == 0 launches nothing.
 * esmb200_knn_scratch_bytes writes the size to *out; it refuses (ESMB200_EINVAL) k or splits out of range, Q < 0 and
 * a NULL out. */
int esmb200_knn_scratch_bytes(int32_t Q, int32_t k, int32_t splits, size_t* out);
int esmb200_knn_search(const void* queries, int64_t q_ld, int32_t Q, const void* base, int64_t b_ld, int64_t N,
                       int32_t D, const float* beta, float alpha, int64_t self_offset, int32_t k, int32_t splits,
                       void* scratch, size_t scratch_bytes, float* out_scores, int64_t* out_idx, void* stream);

/* Streamed k-nearest-neighbour search over a database that arrives in chunks (esm_b200/search.py ShardedIndex).
 * esmb200_knn_search_accumulate: base fp16 [n, b_ld] holds the database's global rows [row0, row0 + n); everything else
 * is as for esmb200_knn_search, with j the global index and self_offset in global rows (query i leaves out global row
 * i + self_offset). keys uint64 [Q, k] (device, dense) is the running list of each query: the top k so far as ranking
 * keys (ord(s) << 32) | (2^32 - 1 - j), descending, 0 for an empty slot (all zeros before the first chunk). The call
 * folds the chunk's candidates into it in place, so after every chunk has been passed once, in any order and any
 * split into chunks, keys hold the same top k esmb200_knn_search returns over the whole database. The chunk may hold
 * fewer than k candidates. Two launches: the fused GEMM + top-k over `splits` stripes, its thresholds seeded with
 * each query's running k-th key, then a merge of the stripe lists with the running list. scratch as
 * esmb200_knn_scratch_bytes(Q, k, splits). 1 <= k <= 128, Q >= 0, n >= 1, row0 >= 0 and row0 + n < 2^31, D, q_ld,
 * b_ld, splits and the alignments as for esmb200_knn_search, keys non-NULL and 8-byte aligned, else ESMB200_EINVAL
 * before any launch. Q == 0 launches nothing.
 * esmb200_knn_decode: keys [Q, k] to out_scores fp32 [Q, k] and out_idx int64 [Q, k] (device, dense), exactly as
 * esmb200_knn_search writes them (an empty slot decodes to NaN and index 2^32 - 1). Q >= 0, 1 <= k <= 128, non-NULL
 * pointers, keys and out_idx 8-byte aligned and out_scores 4-byte aligned, else ESMB200_EINVAL before any launch;
 * Q == 0 launches nothing. One launch. */
int esmb200_knn_search_accumulate(const void* queries, int64_t q_ld, int32_t Q, const void* base, int64_t b_ld,
                                  int64_t n, int64_t row0, int32_t D, const float* beta, float alpha,
                                  int64_t self_offset, int32_t k, int32_t splits, void* scratch, size_t scratch_bytes,
                                  uint64_t* keys, void* stream);
int esmb200_knn_decode(const uint64_t* keys, int32_t Q, int32_t k, float* out_scores, int64_t* out_idx, void* stream);

/* Range search over embeddings (esm_b200/search.py EmbeddingIndex.range_search, ShardedIndex.range_search): every
 * candidate at or above a threshold instead of the top k. The score s(i, j) and the candidates are
 * esmb200_knn_search_accumulate's (global index j = row0 + the chunk row, query i leaves out global row i + self_offset
 * when self_offset >= 0, -0 taken as +0). Candidate j is a hit of query i iff s(i, j) >= tau[i] (tau fp32 [Q], device,
 * never NaN; -0 is taken as +0; -inf makes every candidate a hit). A cosine search passes the smallest fp32 at or
 * above its min_score; an l2 search passes, per query, the smallest fp32 s whose distance sqrt(max(|q|^2 - s, 0))
 * (fp32, correctly rounded) is at most max_distance: the distance does not increase with s, so that is the hit set.
 * esmb200_knn_range: appends the chunk's hits, unordered, to hit_keys uint64 [hit_cap] (the ranking keys
 *   (ord(s) << 32) | (2^32 - 1 - j)) and hit_rows int32 [hit_cap] (the query row), at positions taken from *hit_total
 *   (uint64, device), and adds each query's hits to hit_counts uint64 [Q] (device). Both counters count every hit,
 *   but a hit is written only below hit_cap, so after an overflow they give each query's exact count and the exact
 *   total (set them to 0 before the first chunk; hit_cap 0 with NULL buffers only counts). Chunks are appended one
 *   after another into the same buffers, in any order. One launch: knn_topk_kernel in range mode (fixed thresholds,
 *   a full queue flushed with one global atomicAdd per row), 12 bytes of buffer per hit. No scratch. Q >= 0, n >= 1,
 *   row0 >= 0 and row0 + n < 2^31, D, q_ld, b_ld, splits and the query and base alignments as for
 *   esmb200_knn_search, 0 <= hit_cap < 2^31, non-NULL tau, hit_counts and hit_total (hit_keys and hit_rows too when
 *   hit_cap > 0), 4-byte aligned beta, tau and hit_rows and 8-byte aligned hit_keys, hit_counts and hit_total, else
 *   ESMB200_EINVAL before any launch. Q == 0 launches nothing.
 * esmb200_knn_range_finish: the hits of one range search to CSR. keys and rows hold all nnz = sum(counts) hits, sorted
 *   by query row ascending and, within a query, by key descending (a stable sort by key descending, then a stable sort
 *   by row, leaves them so; keys are distinct within a query, so any correct sort gives the same bits). Writes lims
 *   int64 [Q + 1] (lims[q + 1] - lims[q] = min(counts[q], max_hits), max_hits = -1 for no cap), and each query's
 *   first hits, decoded, to scores fp32 [lims[Q]] and idx int64 [lims[Q]]. scratch:
 *   esmb200_knn_range_finish_scratch_bytes(Q) bytes, 8-byte aligned. Q >= 0, 0 <= nnz < 2^31, max_hits >= 1 or -1,
 *   non-NULL counts, scratch and lims (keys, rows, scores and idx too when nnz > 0), the alignments of their types
 *   and enough scratch, else ESMB200_EINVAL before any launch. Two launches (one when nnz == 0).
 * esmb200_knn_range_finish_scratch_bytes writes (Q + 1) * 8 to *out; it refuses Q < 0 and a NULL out. */
int esmb200_knn_range(const void* queries, int64_t q_ld, int32_t Q, const void* base, int64_t b_ld, int64_t n,
                      int64_t row0, int32_t D, const float* beta, float alpha, int64_t self_offset, const float* tau,
                      int32_t splits, uint64_t* hit_keys, int32_t* hit_rows, int64_t hit_cap, uint64_t* hit_counts,
                      uint64_t* hit_total, void* stream);
int esmb200_knn_range_finish_scratch_bytes(int32_t Q, size_t* out);
int esmb200_knn_range_finish(const uint64_t* keys, const int32_t* rows, int64_t nnz, const uint64_t* counts, int32_t Q,
                             int64_t max_hits, void* scratch, size_t scratch_bytes, int64_t* lims, float* scores,
                             int64_t* idx, void* stream);

/* Inverted-file (IVF) search (esm_b200/search.py IVFIndex). The stored rows fp16 [N, b_ld] (device, 16-byte aligned) are
 * grouped into nlist lists: list l is rows [offsets[l], offsets[l+1]) (offsets int64 [nlist + 1], 0 = offsets[0] <=
 * ... <= offsets[nlist] = N), and ids int64 [N] holds each stored row's original index (distinct, in [0, 2^31)). beta
 * fp32 [N] (or NULL) is in stored order. For each query row i (queries fp16 [Q, q_ld]) the result is the exact top k of
 *     s(i, j) = alpha * (queries_i . rows_j) + beta[j]      (fp32 accumulation of the fp16 products)
 * over the stored rows j of the lists query i probes, leaving out the row with ids[j] == self_ids[i] (self_ids int64
 * [Q], or NULL for none), ranked by (score descending, ids[j] ascending): out_scores fp32 [Q, k] and out_idx int64
 * [Q, k] (= ids[j]), dense. Slots past the probed lists' candidates are score NaN and index -1.
 *   nprobe < nlist: probes int32 [Q, nprobe] (device) names the lists of each query, 1 <= nprobe <= 128; an entry
 *     outside [0, nlist), or one that repeats an earlier entry of its row, probes nothing, so each list is scanned
 *     at most once per query.
 *   nprobe == nlist: every list, probes NULL; the result is then esmb200_knn_search's over the rows in original order,
 *     bit for bit.
 * The scores are esmb200_knn_search's, so a query's result depends only on the query, the rows and its probed lists:
 * not on the other queries, Q or the launch configuration.
 * Work: the (query, probe) pairs are grouped by list (probed only: a count, a scan, the placement, the work items and a
 * gather of the query rows into scratch, then one device-to-host read of the work-item count, the call's only host
 * synchronisation); one knn_topk_kernel<false, true> CTA per work item (a list, a block of <= 64 queries probing it,
 * a stripe of T of its 256-row tiles), so each list is read once per query block; then a merge of each query's
 * partial lists. Stripes: probed, T = ceil((ceil(N / 256) + nlist) / 64), so a query has at most nprobe + 64 partial
 * lists; every list, the rows split into min(ceil(N / 256), ceil(264 / ceil(Q / 64))) stripes (about two waves of a
 * 132-SM H100).
 * scratch: esmb200_ivf_scratch_bytes(Q, nprobe, nlist, N, D, k) bytes, 256-byte aligned; it grows with Q: about
 * Q * nprobe * D * 2 bytes of gathered query rows and Q * (nprobe + 64) * k * 8 of partial lists (probed). 1 <= k <= 128,
 * 1 <= N < 2^31, Q >= 0, 1 <= nlist <= min(N, 2^24), nprobe as above with Q * nprobe < 2^30 and Q * R < 2^31 (R the
 * partial lists per query: nprobe + 64, or the stripe count when every list is probed), D % 64 == 0, q_ld and b_ld
 * >= D and multiples of 8, probes NULL exactly when nprobe == nlist, non-NULL queries, rows, ids, offsets, scratch and
 * outputs with their alignments and enough scratch, else ESMB200_EINVAL before any launch. Q == 0 launches nothing.
 * A work-item count past the bound (offsets that do not partition [0, N); offsets are not otherwise checked) is
 * refused after the grouping launches, before the scan. esmb200_ivf_scratch_bytes writes the size to *out, with the same refusals. */
int esmb200_ivf_scratch_bytes(int32_t Q, int32_t nprobe, int32_t nlist, int64_t N, int32_t D, int32_t k, size_t* out);
int esmb200_ivf_search(const void* queries, int64_t q_ld, int32_t Q, const void* rows, int64_t b_ld, int64_t N,
                       const int64_t* ids, const int64_t* offsets, int32_t nlist, int32_t D, const float* beta,
                       float alpha, const int32_t* probes, int32_t nprobe, const int64_t* self_ids, int32_t k,
                       void* scratch, size_t scratch_bytes, float* out_scores, int64_t* out_idx, void* stream);

/* k-means centroid means, exactly (esm_b200/search.py IVFIndex training). rows fp16 [n, ld] (device, 16-byte aligned,
 * first D columns), assign int64 [n] (a row with assign outside [0, nlist) is left out). Every fp16 value is an integer
 * multiple of 2^-24, so
 *     sums[c, j]  = sum over rows r with assign[r] == c of rows[r, j] * 2^24      (int64, exact)
 *     counts[c]   = the rows with assign == c                                     (int64)
 *     means[c, j] = fp32(((double)sums[c, j] / counts[c]) * 2^-24), 0 for an empty cluster
 * are IEEE-defined and do not depend on the order of the additions (atomics). sums int64 [nlist, D], means_out fp32
 * [nlist, D] and counts_out int64 [nlist] (device, dense) are outputs. n <= 2^23 (|x| <= 65504, so |sums| < 2^63),
 * D % 8 == 0, ld >= D a multiple of 8, 1 <= nlist <= 2^24, non-NULL and aligned pointers, else ESMB200_EINVAL before
 * any launch. Two memsets and two launches. */
int esmb200_kmeans_means(const void* rows, int64_t ld, int64_t n, int32_t D, const int64_t* assign, int32_t nlist,
                         int64_t* sums, float* means_out, int64_t* counts_out, void* stream);

/* Pairwise alignment of proteins by their per-residue embeddings (esm_b200/align.py; the EBA / pLM-BLAST family of
 * methods). A new operation with no reference code. Pair p (of P) has La query rows and Lb target rows, La, Lb >= 1:
 * query rows [q_off[p], q_off[p+1]) and target rows [t_off[p], t_off[p+1]), its similarity S' as [La, Lb] fp32
 * row-major at s_off[p] (offsets: int64 [P+1] device arrays from 0, non-decreasing; n_q = q_off[P] query rows,
 * n_t = t_off[P] target rows and n_cells = s_off[P] are passed from the host as well; the per-pair offsets are
 * checked by the caller). Results depend only on the pair: not on the other pairs, their order or the device.
 * esmb200_align_similarity: q_rows, t_rows fp16 [*, D] (16-byte aligned, D % 64 == 0, rows normalised and
 *   zero-padded by the caller), S[i,j] = q_i . t_j with fp32 accumulation of the fp16 products (mma.sync).
 *   zscore 1: S'[i,j] = 0.5 * ((S - mu_r_i) / sd_r_i + (S - mu_c_j) / sd_c_j), mean and population standard
 *   deviation of row i and column j taken in fp64 in a fixed order and rounded to fp32, a term 0 where its sd is 0;
 *   zscore 0: S' = S. Written to out at s_off. The z-score statistics use the scratch.
 * esmb200_align: the affine-gap dynamic programme on S' in fp32, gap_open o >= 0 and gap_extend e >= 0 finite:
 *     E[i][j] = max(H[i][j-1] - o, E[i][j-1] - e)   target residue j against a gap, op 'T'
 *     F[i][j] = max(H[i-1][j] - o, F[i-1][j] - e)   query residue i against a gap,  op 'Q'
 *     H[i][j] = max(H[i-1][j-1] + S'[i-1][j-1], E[i][j], F[i][j] [, 0 local])       diagonal,  op 'M'
 *   one fp32 add or subtract per candidate, no fused operations. ESMB200_ALIGN_LOCAL: H = 0 on row 0 and column 0,
 *   E = F = -inf there; the end cell is the largest H, a tie to the smallest i, then j (a score of 0 ends at (0, 0)).
 *   ESMB200_ALIGN_GLOBAL: H[0][0] = 0, row 0 and column 0 follow the same recurrences without the diagonal and with
 *   -inf outside the matrix; the end cell is (La, Lb). The source of a value is the first candidate equal to the
 *   maximum in the order diagonal, E, F, zero (H) and open, extend (E, F). Traceback from the end cell in state H:
 *   diagonal emits M to (i-1, j-1); E or F switches state at the same cell; E emits T to (i, j-1) and F emits Q to
 *   (i-1, j), into state H if it opened and its own state if it extended. Local stops at a cell whose H came from
 *   zero or at row or column 0; global at (0, 0).
 *   Outputs (device): scores fp32 [P]; spans int32 [P, 4] = q0, q1, t0, t1 (0-based, end exclusive); the op string
 *   of pair p in query->target order at ops + q_off[p] + t_off[p] (La + Lb bytes per pair, n_q + n_t in all);
 *   n_ops int32 [P]. Two kernels: one warp per pair runs the wavefront and stores one direction byte per cell, then one
 *   thread per pair walks the traceback.
 * scratch: esmb200_align_scratch_bytes(P, n_q, n_t, n_cells) bytes, 256-byte aligned, for either call: about one byte
 *   per cell plus 32 per row and column and 8 per row and column (border rows of the programme, z-score statistics);
 *   0 for a negative argument. Refused with ESMB200_EINVAL before any launch: P < 0, n_q, n_t or n_cells < P,
 *   n_cells > 2^40, D, an unknown mode or zscore, non-finite or negative penalties, NULL pointers, unaligned or too
 *   little scratch ("more cells than the scratch"). P == 0 launches nothing. No atomics. */
#define ESMB200_ALIGN_LOCAL 0
#define ESMB200_ALIGN_GLOBAL 1
size_t esmb200_align_scratch_bytes(int32_t P, int64_t n_q, int64_t n_t, int64_t n_cells);
int esmb200_align_similarity(const void* q_rows, const void* t_rows, int32_t D, const int64_t* q_off,
                             const int64_t* t_off, const int64_t* s_off, int32_t P, int64_t n_q, int64_t n_t,
                             int64_t n_cells, int32_t zscore, float* out, void* scratch, size_t scratch_bytes,
                             void* stream);
int esmb200_align(const float* s, const int64_t* q_off, const int64_t* t_off, const int64_t* s_off, int32_t P,
                  int64_t n_q, int64_t n_t, int64_t n_cells, int32_t mode, float gap_open, float gap_extend,
                  void* scratch, size_t scratch_bytes, float* scores, int32_t* spans, uint8_t* ops, int32_t* n_ops,
                  void* stream);

/* ---- single-kernel entry points (used by the parity tests and profiles; same kernels as above) ---- */

/* out = epilogue(A[M,K] fp16 x W[N,K]^T fp16 + bias[N]);  epilogue: 0 qkv+rope -> fp16, 1 residual-add into fp32 out,
 * 2 gelu -> fp16, 3 fp32, 4 gelu -> fp32. rope_* / T / E only for epilogue 0. K % 8 == 0; N % 64 == 0 for an fp16
 * output (epilogues 0, 2), N % 32 == 0 for an fp32 one. */
int esmb200_gemm_f16(int32_t epilogue, const void* a_f16, const void* w_f16, const float* bias, void* out, int32_t M,
                     int32_t N, int32_t K, const float* rope_cos, const float* rope_sin, int32_t T, int32_t E,
                     void* stream);

/* qkv[M,3E] fp16 = A[M,E] fp16 x [Wq;Wk;Wv]^T + bias, q columns scaled by q_scale, q/k rotated when rope tables are
 * given (ESM-2: multihead_attention.py:258-261,354-355) or left unrotated when rope_cos == rope_sin == NULL (MSA axial
 * attention: axial_attention.py:79-81 with q_scale = d^-1/2 / sqrt(rows), :199-202 with q_scale = d^-1/2). */
int esmb200_gemm_qkv_f16(const void* a_f16, const void* w_qkv_f16, const float* bias_qkv, void* out_f16, int32_t M,
                         int32_t E, float q_scale, const float* rope_cos, const float* rope_sin, int32_t T,
                         void* stream);

/* The layer's QKV projection at any head width: qkv = [q*q_scale | k | v] in head slots, q/k rotated when tables are
 * given. d = E / H, slots = 1 (d <= 64) or 2 (d <= 128), Ea = 64 * slots * H; w [3Ea, K] packed by head_slot (row
 * s*Ea + slot column of projection output h*d + j, zero rows elsewhere; DESIGN.md section 1).
 * precision 0: a fp16 [M,E], w fp16 [3Ea,E]            -> fp16 [M,3Ea]
 *           1: a [M,2E] hi|lo, w [3Ea,2E] hi|lo         -> [M,6Ea] hi|lo
 *           2: a e4m3 [M,E] + a_scales, w e4m3 + w_scales -> fp16 [M,3Ea]
 * rope tables [T, 32*slots] or both NULL. The same launch as the layers' QKV projection; refuses the widths and
 * precisions esmb200_layer_create refuses. */
int esmb200_gemm_qkv_heads(int32_t precision, const void* a, const float* a_scales, const void* w,
                           const float* w_scales, const float* bias, void* out, int32_t M, int32_t E, int32_t H,
                           float q_scale, const float* rope_cos, const float* rope_sin, int32_t T, void* stream);

/* ctx[B*T,E] fp16 = softmax(q k^T + key padding mask) v per head, from qkv fp16 [B*T,3E] (q pre-scaled, q/k rotated).
 * scratch: at least esmb200_attention_scratch_bytes(B,T). attn_probs as in esmb200_layer_forward. */
size_t esmb200_attention_scratch_bytes(int32_t B, int32_t T);
int esmb200_attention(const void* qkv_f16, const uint8_t* pad_mask, void* ctx_f16, float* attn_probs, int32_t B,
                      int32_t T, int32_t H, void* scratch, void* stream);
/* The same for head_dim 128 (esm2_t48_15B, esm/pretrained.py:390-397): qkv fp16 [B*T, 3*128*H], ctx fp16 [B*T, 128*H];
 * a head is two adjacent 64-wide column slots (DESIGN.md section 1), any fixed permutation of the 128 dimensions that is
 * shared by q, k and v gives the same result. */
int esmb200_attention128(const void* qkv_f16, const uint8_t* pad_mask, void* ctx_f16, float* attn_probs, int32_t B,
                         int32_t T, int32_t H, void* scratch, void* stream);

/* ---- MSA Transformer axial attention on qkv fp16 [B*R*C, 3E] (B alignments, R rows, C columns; q pre-scaled) ----
 * esmb200_tied_row_attention: RowSelfAttention.compute_attention_weights / compute_attention_update,
 *   esm/axial_attention.py:71-111 — logits summed over the R rows (:87), key_pad [B,C] (1 = padded key column, filled
 *   with -10000, :94-97; NULL = none), softmax over the key columns (:105), ctx[B*R*C,E] fp16 = P v per row (:108).
 *   The caller zeroes q at padded positions (:82-85). attn_probs: optional fp32 [H,B,C,C] (the reference's return
 *   layout), NULL to skip. scratch: esmb200_tied_row_attention_scratch_bytes(B,C,H). C <= 1024.
 * esmb200_column_attention: ColumnSelfAttention.compute_attention_update, esm/axial_attention.py:182-222 — per
 *   alignment column, attention over the R rows; pad_mask [B*C, R] (1 = padded key; such keys get probability 0 where
 *   the reference fills -10000, identical unless every key of a column is padded), ctx[B*R*C,E] fp16.
 *   scratch: esmb200_attention_scratch_bytes(B*C, R). */
size_t esmb200_tied_row_attention_scratch_bytes(int32_t B, int32_t C, int32_t H);
int esmb200_tied_row_attention(const void* qkv_f16, const uint8_t* key_pad, void* ctx_f16, float* attn_probs, int32_t B,
                               int32_t R, int32_t C, int32_t H, void* scratch, size_t scratch_bytes, void* stream);
int esmb200_column_attention(const void* qkv_f16, const uint8_t* pad_mask, void* ctx_f16, int32_t B, int32_t R,
                             int32_t C, int32_t H, void* scratch, void* stream);

/* n_layers x AxialTransformerLayer.forward (esm/modules.py:195-221) = the layer loop of MSATransformer.forward
 * (esm/model/msa_transformer.py:190-201), in place on the batch-major residual stream x [B,R,C,E] fp32:
 *   x += out_proj(tied_row_attention(LN(x)));  x += out_proj(column_attention(LN(x)));  x += fc2(gelu(fc1(LN(x))))
 * row_layers[i]: an esmb200_layer created with fc1_weight == NULL (attention-only) from row_self_attention's
 *   layer_norm + q/k/v/out projections; col_layers[i]: column_self_attention's layer_norm + projections as ln1/q/k/v/out
 *   and feed_forward_layer's layer_norm + fc1/fc2 as ln2/fc1/fc2.
 * pad_mask [B,R,C] and col_pad_mask [B,C,R] (its transpose): 1 = padding, both NULL for unpadded alignments. As in
 *   the reference (axial_attention.py:82-97), the row attention zeroes q at every padded token, and its padded key
 *   columns are those of row 0 of each alignment (pad_mask[b, 0, :]).
 * row_attn_out: NULL, or n_layers pointers (NULL entries allowed) to fp32 [H,B,C,C] buffers (the reference's
 *   row-attention return layout, axial_attention.py:87,105).
 * col_attn_out: NULL, or n_layers pointers (NULL entries allowed) to fp32 [B*C,H,R,R] buffers: the column-attention
 *   probabilities of alignment column c of alignment b at [b*C + c] (the reference returns them as [H,C,B,R,R],
 *   axial_attention.py:206,216). Any B*C*H: the probability kernel runs one launch per 65535 / H column
 *   sequences. x and the row maps are the same bits with and without them.
 * workspace: esmb200_axial_workspace_bytes(E,F,B,R,C) bytes, or esmb200_axial_workspace_bytes_split(E,F,B,R,C) for
 *   layers created with precision = 1 (fp32x3: the activations, qkv, ctx and P are stored as fp16 hi | lo pairs).
 *   All 2 * n_layers layers must share one precision; mixed precision is ESMB200_EINVAL. */
size_t esmb200_axial_workspace_bytes(int32_t E, int32_t F, int32_t B, int32_t R, int32_t C);
size_t esmb200_axial_workspace_bytes_split(int32_t E, int32_t F, int32_t B, int32_t R, int32_t C);
int esmb200_axial_stack_forward(esmb200_layer* const* row_layers, esmb200_layer* const* col_layers, int32_t n_layers,
                                float* x, const uint8_t* pad_mask, const uint8_t* col_pad_mask, int32_t B, int32_t R,
                                int32_t C, float* const* row_attn_out, float* const* col_attn_out, void* workspace,
                                size_t workspace_bytes, void* stream);

/* MSA Transformer embedding prologue, esm/model/msa_transformer.py:155-172 (+ LearnedPositionalEmbedding.forward,
 * esm/modules.py:241-257): x[B,R,C,E] fp32 = LayerNorm(embed_tokens[tok] + embed_positions[pos] +
 * msa_position_embedding[r]) * (1 - is_pad). tokens int64 [B,R,C]; pos_table [max_positions + padding_idx + 1, E];
 * msa_pos [>=R, msa_pos_dim] or NULL, msa_pos_dim = E or 1 (the initial esm_msa1 release, pretrained.py:123-125).
 * E % 4 == 0, E <= 2560, C <= 12288 (one alignment row's positions are held in shared memory). */
int esmb200_msa_embed(const int64_t* tokens, const float* embed_table, const float* pos_table, const float* msa_pos,
                      int32_t msa_pos_dim, const float* ln_weight, const float* ln_bias, float eps, float* x,
                      int32_t B, int32_t R, int32_t C, int32_t E, int32_t padding_idx, void* stream);

/* Contact head, one layer's share (ContactPredictionHead.forward esm/modules.py:338-357, symmetrize :27-29, apc :32-41):
 * attn = that layer's attention maps fp32 [B,H,T,T] (batch_stride floats between batch elements, so a slice of a stacked
 * [B,L,H,T,T] tensor works), cropped to positions [lo,hi) and multiplied by keep[b,i]*keep[b,j] (keep [B,T], 1 = not
 * <eos>; NULL = no masking). S = hi - lo.
 *   acc      [B,S,S]            += sum_h w[h] * A_h   (zeroed by the caller before the first layer)
 *   row_sum  [B,H,S]             = rowsum(A_h)
 *   col_part [B,H,ceil(S/16),S]  = column sums of each 16-row stripe; colsum(A_h) = sum over the stripe axis
 * No atomics: results are bit-reproducible. a1_c = row_sum + colsum feeds esmb200_contact_finalize. */
int esmb200_contact_accumulate(const float* attn, int64_t batch_stride, const float* w, const uint8_t* keep, float* acc,
                               float* row_sum, float* col_part, int32_t B, int32_t H, int32_t T, int32_t lo, int32_t hi,
                               void* stream);

/* Contact head tail (modules.py:33-41,352-357): out[b,i,j] = sigmoid(acc[b,i,j] + acc[b,j,i] - sum_c u[b,c,i]*a1[b,c,j] + bias)
 * with a1 [B,C,S] (C = layers*heads channels) and u = a1 * w_c / sum_i a1_c[i] prepared by the caller; bias = device
 * pointer to one float or NULL; out [B,S,S]. */
int esmb200_contact_finalize(const float* acc, const float* u, const float* a1, const float* bias, float* out, int32_t B,
                             int32_t C, int32_t S, void* stream);

/* fp32 [M,E] -> LayerNorm -> fp16 [M,E] (the GEMM A operand) */
int esmb200_layernorm_f16(const float* x, const float* weight, const float* bias, void* out_f16, int32_t M, int32_t E,
                          float eps, void* stream);

/* ---- launch accounting and per-launch timing (bench.py roofline numbers) ----
 * esmb200_launch_count: kernels launched by this library since it was loaded.
 * esmb200_profile_enable(n): n > 0 brackets each of the next n launches with CUDA events on the launch stream
 *   (0 disables and frees the events); esmb200_profile_read returns up to max_records (tag, milliseconds) pairs,
 *   synchronising on the recorded events, and resets the record list.
 *   tags: 0 LN1->f16, 1 QKV+RoPE GEMM, 2 attention, 3 out-proj GEMM, 4 LN2->f16, 5 fc1+GELU GEMM, 6 fc2 GEMM,
 *         7 key bits, 8 embed, 9 LayerNorm fp32, 10 attention probs, 11 convert, 12 other GEMM, 13 mean pool,
 *         14 tied row logits, 15 tied row softmax, 16 tied row update, 17 log_softmax rows (variant scoring),
 *         18 window merge, 19 categorical Jacobian contacts (each of its kernels), 20 sampling (esmb200_sample_order
 *         and each kernel of esmb200_sample_rows), 21 greedy MSA row selection (each kernel of
 *         esmb200_msa_greedy_select), 22 nearest-neighbour search (each kernel of esmb200_knn_search,
 *         esmb200_knn_search_accumulate, esmb200_knn_decode, esmb200_ivf_search and esmb200_kmeans_means),
 *         23 embedding alignment (each kernel of esmb200_align_similarity and esmb200_align) */
long long esmb200_launch_count(void);
int esmb200_profile_enable(int32_t max_launches);
int esmb200_profile_read(int32_t* tags, float* ms, int32_t max_records);

/* ---- fp8 precision building blocks (e4m3 operands, power-of-two scales s: q = e4m3_rn(x / s), x ~ q * s; s is the
 * smallest power of two with amax / s <= 448 over its block, at least 2^-126, and 1 for an all-zero block; a partial
 * block takes its amax over its valid elements). Used by the fp8 layers and kernel-level tests.
 * esmb200_layernorm_fp8: fp32 [M,E] -> LayerNorm -> e4m3 [M,E] + scales [ceil(E/128), M] (scales[kb * M + row]).
 * esmb200_quantize_fp8:  fp32 [rows,K] -> e4m3 [rows,K]; block_rows 1: scales [ceil(K/128), rows] as above;
 *                        block_rows 128 (weights): scales [ceil(rows/128), ceil(K/128)]. Deterministic.
 * esmb200_gemm_fp8:      A [M,K] e4m3 with 1 x 128 scales (a_scales [ceil(K/128), M]), W [N,K] e4m3 with 128 x 128
 *                        scales (w_scales [ceil(N/128), ceil(K/128)]), fp32 accumulation promoted per 128-wide K block.
 *                        epilogue 0: qkv + rope -> fp16 [M,N] as esmb200_gemm_f16 (q_scale 0.125, N == 3E);
 *                        1: out fp32 [M,N] += y + bias (N % 32 == 0); 5: erf-GELU(y + bias) -> e4m3 [M,N] with
 *                        out_scales [N/128, M] (N % 128 == 0). K % 16 == 0. */
int esmb200_layernorm_fp8(const float* x, const float* weight, const float* bias, void* out_e4m3, float* scales,
                          int32_t M, int32_t E, float eps, void* stream);
int esmb200_quantize_fp8(const float* src, void* dst_e4m3, float* scales, int32_t rows, int32_t K, int32_t block_rows,
                         void* stream);
int esmb200_gemm_fp8(int32_t epilogue, const void* a_e4m3, const float* a_scales, const void* w_e4m3,
                     const float* w_scales, const float* bias, void* out, float* out_scales, int32_t M, int32_t N,
                     int32_t K, const float* rope_cos, const float* rope_sin, int32_t T, int32_t E, void* stream);

/* fp32 -> fp16 elementwise */
int esmb200_convert_f16(const float* src, void* dst_f16, size_t n, void* stream);

/* ---- fp32x3 precision building blocks (operands as fp16 hi | lo pairs along K): the LM head, the MSA layer's
 * attention-map path (esm_b200/msa.py) and kernel-level tests.
 * esmb200_layernorm_split: fp32 [M,E] -> LayerNorm -> fp16 [M,2E] (hi in columns [0,E), lo = rn(y - hi) in [E,2E)).
 * esmb200_convert_split:   fp32 [rows,K] -> fp16 [rows,2K] the same way (weights).
 * esmb200_gemm_split:      esmb200_gemm_f16 with a [M,2K], w [N,2K]; fp16 outputs (QKV_ROPE, BIAS_GELU) are written as
 *                          [M,2N] hi | lo, fp32 outputs as [M,N].  K % 64 == 0.
 * esmb200_attention_split: esmb200_attention on qkv [B*T, 6E] = [q k v]_hi | [q k v]_lo -> ctx [B*T, 2E] hi | lo.
 * esmb200_gemm_qkv_split:  esmb200_gemm_qkv_f16 without rope tables (the MSA axial attention): a [M,2E], w_qkv [3E,2E]
 *                          (esmb200_convert_split of [Wq;Wk;Wv]), q columns scaled by q_scale -> qkv [M,6E] hi | lo.
 *                          E % 64 == 0.
 * esmb200_tied_row_attention_split: esmb200_tied_row_attention on qkv [B*R*C, 6E] -> ctx [B*R*C, 2E] hi | lo; the
 *                          logits sum each alignment row's 64-wide slab in a fresh fp32 fragment; attn_probs as in
 *                          the fp16 call. The caller zeroes q_hi AND q_lo at padded positions. scratch:
 *                          esmb200_tied_row_attention_split_scratch_bytes(B,C,H) (P is stored as hi | lo).
 * esmb200_column_attention_split: esmb200_column_attention on qkv [B*R*C, 6E] -> ctx [B*R*C, 2E] hi | lo; scratch:
 *                          esmb200_attention_scratch_bytes(B*C, R). */
int esmb200_layernorm_split(const float* x, const float* weight, const float* bias, void* out_f16, int32_t M, int32_t E,
                            float eps, void* stream);
int esmb200_convert_split(const float* src, void* dst_f16, int64_t rows, int32_t K, void* stream);
int esmb200_gemm_split(int32_t epilogue, const void* a, const void* w, const float* bias, void* out, int32_t M,
                       int32_t N, int32_t K, const float* rope_cos, const float* rope_sin, int32_t T, int32_t E,
                       void* stream);
int esmb200_attention_split(const void* qkv, const uint8_t* pad_mask, void* ctx, float* attn_probs, int32_t B, int32_t T,
                            int32_t H, void* scratch, void* stream);
int esmb200_gemm_qkv_split(const void* a, const void* w_qkv, const float* bias_qkv, void* out, int32_t M, int32_t E,
                           float q_scale, void* stream);
size_t esmb200_tied_row_attention_split_scratch_bytes(int32_t B, int32_t C, int32_t H);
int esmb200_tied_row_attention_split(const void* qkv, const uint8_t* key_pad, void* ctx, float* attn_probs, int32_t B,
                                     int32_t R, int32_t C, int32_t H, void* scratch, size_t scratch_bytes,
                                     void* stream);
int esmb200_column_attention_split(const void* qkv, const uint8_t* pad_mask, void* ctx, int32_t B, int32_t R, int32_t C,
                                   int32_t H, void* scratch, void* stream);

/* ---- process-wide launch knobs (A/B measurements; the defaults are the product configuration) ----
 * "pdl"       0 (default) | 1: programmatic dependent launch between the layer's kernels        env ESMB200_PDL
 * Returns ESMB200_EINVAL for an unknown name or value. Not thread-safe against concurrent launches. */
int esmb200_set_option(const char* name, int32_t value);

#ifdef __cplusplus
}
#endif
#endif /* ESMB200_H_ */
