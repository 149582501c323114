"""float64 references of single kernels, shared by the kernel-level GPU tests and checked on the CPU by
tests/test_kernel_refs_host.py (so that a wrong reference cannot make a GPU test pass).

  * contact_partials: the accumulators of the fused probability + contact pass (csrc/attention_contact.cuh) in the
    kernel's own layout: acc [B,S,S], row_part / col_part [B,H,4*ceil(T/128),S], one partial per 32-key / 32-query
    quarter of each 128-wide tile;
  * gemm_launches: every (epilogue, N, K) GEMM a model's forward launches (api.cu attention_block / ffn_block, the LM
    head of model.py RobertaLMHead.forward_native, the MSA Transformer's layer in msa.py);
  * gemm_exact / gemm_acc_bound / f16_bound / residual_bound / qkv_ref / qkv_bound: the fp16 GEMM's float64 reference
    and the bounds of its epilogues (residual add, q scale and RoPE);
  * slot_columns / slot_rows / rope_pair_sum / qkv_ref_heads: heads of any width in zero-padded 64-wide slots, mapped
    from the reference's rotate-half pairing, and the QKV projection in the reference's layout at any head width;
  * gelu_bound: the error bound of the GEMM epilogue's erf-GELU (csrc/gemm_common.cuh gelu_erf);
  * split16 / join64 / split_rep_bound / split_acc_bound / FP32X3_MODELS: the fp32x3 precision's hi | lo operand pairs,
    the bound of their representation, the accumulation bound of the three-pass split GEMM and the models it runs;
  * attention64 / attention64_rows / attn_ctx_bound / attn_relfro_gate / attn_probs_bound / attn_rowsum_bound /
    attn_max_bound / attn_sum_bound: float64 softmax attention on fp16 q, k, v (whole heads, or slices of their query
    rows so that T = 16384 fits a few GB) and the first-order error model of the fp16 attention kernels
    (csrc/attention_wg.cuh, attention8.cuh <false, 2>, attention_probs.cuh modes 0 and 2);
  * tied64 / tied_softmax64 / tied_probs_bound / tied_P_bound / tied_rowsum_bound / tied_pv / tied_ctx_bound /
    tied_relfro_gate: the MSA Transformer's tied row attention (csrc/tied_attention.cuh, fp16 and fp32x3) end to end
    and stage by stage, each stage on the kernel's own inputs (logits, softmax of its logits, P V of its P);
  * positions / embed_esm2_64 / embed_esm1b_64 / embed_msa_64 / embed_scale_bound / ln_tol / ln_scale: the three
    embedding prologues (csrc/elementwise.cuh embed_tokens_kernel, esm1b_embed_kernel, msa_embed_kernel);
  * mean_pool64 / mean_pool_bound, log_softmax64 / log_softmax_bound: the per-sequence mean representation and the
    log-softmax rows of variant scoring;
  * contact_stripes: the accumulators of the standalone contact pass (contact_accumulate_kernel) in its own layout;
  * layer64: one ESM-2 TransformerLayer in float64 at any even head width.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch

EPI_QKV_ROPE, EPI_BIAS_RESIDUAL, EPI_BIAS_GELU, EPI_BIAS_F32, EPI_BIAS_GELU_F32 = range(5)

U32 = 2.0 ** -24  # unit roundoff of fp32


# ---- contact head ---------------------------------------------------------------------------------------------------
def contact_mask(keep: Optional[torch.Tensor], T: int, lo: int, hi: int, device=None) -> torch.Tensor:
    """[B or 1, T] float64: 1 at positions inside the crop [lo, hi) that are not <eos> (keep = tokens != eos)."""
    crop = torch.zeros(T, dtype=torch.float64, device=device)
    crop[lo:hi] = 1
    if keep is None:
        return crop[None]
    return keep.to(device=device, dtype=torch.float64) * crop[None]


def masked_maps(attn: torch.Tensor, keep: Optional[torch.Tensor], lo: int, hi: int) -> torch.Tensor:
    """attn [B,H,T,T] (one layer) -> float64 A_h with the rows and columns outside the crop or at <eos> zeroed."""
    B, H, T, _ = attn.shape
    m = contact_mask(keep, T, lo, hi, attn.device)
    m = m.expand(B, T)
    return attn.double() * (m[:, None, :, None] * m[:, None, None, :])


def quarter_sums(x: torch.Tensor, dim: int) -> torch.Tensor:
    """Sum `x` over consecutive 32-wide groups along `dim` (padded with zeros to a multiple of 128): the group g holds
    indices [32 g, 32 g + 32), i.e. quarter g % 4 of 128-wide tile g // 4."""
    n = x.shape[dim]
    nt = (n + 127) // 128
    pad = [0, 0] * (x.ndim - 1 - (dim % x.ndim)) + [0, 128 * nt - n]
    xp = torch.nn.functional.pad(x, pad)
    shape = list(xp.shape)
    d = dim % x.ndim
    shape[d:d + 1] = [4 * nt, 32]
    return xp.reshape(shape).sum(d + 1)


def contact_partials(attn: torch.Tensor, w: torch.Tensor, keep: Optional[torch.Tensor], lo: int, hi: int):
    """One layer's share of the fused contact accumulators, float64.
    attn [B,H,T,T], w [H] -> (acc [B,S,S] = sum_h w_h A_h, row_part [B,H,4nt,S], col_part [B,H,4nt,S]) with
    row_part[b,h,4kt+q,i-lo] = sum of A_h[i, j] over the keys j of quarter q of key tile kt, and
    col_part[b,h,4qt+r,j-lo] = sum of A_h[i, j] over the queries i of quarter r of query tile qt."""
    a = masked_maps(attn, keep, lo, hi)
    acc = torch.einsum("bhij,h->bij", a, w.double().to(a.device))[:, lo:hi, lo:hi]
    row = quarter_sums(a, -1)[:, :, lo:hi, :].transpose(-1, -2)  # [B,H,4nt,S]
    col = quarter_sums(a, -2)[:, :, :, lo:hi]                     # [B,H,4nt,S]
    return acc, row, col


def contacts_from_partials(acc: torch.Tensor, row: torch.Tensor, col: torch.Tensor, w: torch.Tensor,
                           bias: Optional[float]) -> torch.Tensor:
    """The contact head from the accumulators of all layers, float64: row/col [L,B,H,4nt,S], w [L,H], acc [B,S,S].
    logit = acc + acc^T - sum_c (w_c / a12_c) a1_c a1_c^T + bias, a1_c = rowsum + colsum (model.py
    ContactPredictionHead.forward)."""
    L, B, H, _, S = row.shape
    a1 = (row.double().sum(3) + col.double().sum(3)).permute(1, 0, 2, 3).reshape(B, L * H, S)
    wl = w.double().reshape(1, L * H, 1).to(a1.device)
    u = a1 * wl / a1.sum(-1, keepdim=True)
    acc = acc.double()
    logits = acc + acc.transpose(-1, -2) - torch.einsum("bci,bcj->bij", u, a1)
    if bias is not None:
        logits = logits + bias
    return torch.sigmoid(logits)


def sum_bound(terms_abs: torch.Tensor, n: int) -> torch.Tensor:
    """Bound of an n-term fp32 recursive sum (any order) of values with absolute sum `terms_abs`: (n - 1) u sum|x|."""
    return (n - 1) * U32 * terms_abs


# ---- fp16 GEMM epilogues (csrc/gemm2.cuh) ---------------------------------------------------------------------------
def gemm_exact(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """(a w^T + bias in float64, sum_k |a_k w_k|) on the kernel's own operands"""
    ad, wd = a.double(), w.double()
    return ad @ wd.t() + bias.double(), ad.abs() @ wd.abs().t()


def gemm_acc_bound(absdot: torch.Tensor, K: int, y: torch.Tensor) -> torch.Tensor:
    """|out - y| of the fp16 GEMM before any epilogue function: the tensor core sums each k16 step's exact products into
    the fp32 accumulator with truncation, (K/16 + 4) 2^-22 sum_k |a_k w_k| (one ulp per step, doubled for slack), plus
    the bias add and the fp32 result (2 u |y|)."""
    return (K / 16 + 4) * 2.0 ** -22 * absdot + 2 * U32 * y.abs()


def f16_bound(y: torch.Tensor) -> torch.Tensor:
    """rounding of a finite fp32 value to fp16: half an ulp, 2^-11 relative, 2^-25 absolute below the normal range."""
    return 2.0 ** -11 * y.abs() + 2.0 ** -25


def residual_bound(acc: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    """|x' - want| for the residual epilogue x' = x + y (EPI_BIAS_RESIDUAL, the fp32 add in the L2), want = x + y64:
    the update's own bound `acc` (gemm_acc_bound, split_acc_bound or fp8_refs.acc_bound) and the fp32 add (u |want|)."""
    return acc + U32 * want.abs()


def qkv_ref(a, w, bias, q_scale, E, T=None, cos=None, sin=None):
    """[q*scale | k | v] in float64 (the bias added before the scale), with rotate-half RoPE on every 64-column group
    of q and k: pair (c, c + 32) rotated by table column c of a [T, 32] table (row r at position r % T).  Returns
    (y, absdot) with absdot the matching sum of |products| (rotated pairs: both members' sums, |cos|, |sin| <= 1)."""
    y, absdot = gemm_exact(a, w, bias)
    y[:, :E] *= q_scale
    absdot[:, :E] *= q_scale
    if cos is not None:
        M = y.shape[0]
        t = torch.arange(M, device=y.device) % T
        c, s = cos.double()[t][:, :32], sin.double()[t][:, :32]
        for g0 in range(0, 2 * E, 64):
            x1, x2 = y[:, g0:g0 + 32].clone(), y[:, g0 + 32:g0 + 64].clone()
            y[:, g0:g0 + 32], y[:, g0 + 32:g0 + 64] = x1 * c - x2 * s, x2 * c + x1 * s
            d1, d2 = absdot[:, g0:g0 + 32].clone(), absdot[:, g0 + 32:g0 + 64].clone()
            absdot[:, g0:g0 + 32] = absdot[:, g0 + 32:g0 + 64] = d1 + d2
    return y, absdot


def slot_columns(d: int, H: int) -> torch.Tensor:
    """[H d] long: the attention-side column of projection output h d + j at head width d.  rotary_embedding.py's
    rotate_half pairs dimension j with j + d/2 under the table column p = j mod d/2; the QKV epilogue rotates columns
    (c, c + 32) of each 64-wide slot by table column 32 (slot mod slots) + c.  So pair p of head h goes to slot p // 32
    of the head's head_slots(H d, H) slots, at columns p % 32 and 32 + p % 32, and meets table column p."""
    slots, half = head_slots(d * H, H), d // 2
    cols = torch.empty(H * d, dtype=torch.long)
    for h in range(H):
        for p in range(half):
            c = (h * slots + p // 32) * 64 + p % 32
            cols[h * d + p], cols[h * d + half + p] = c, c + 32
    return cols


def slot_rows(d: int, H: int) -> torch.Tensor:
    """[3 H d] long: the row of the head-slot-packed [Wq;Wk;Wv] ([3 Ea, K]) that holds each row of the reference's
    [Wq;Wk;Wv], and the column of the kernel's [q | k | v] output ([M, 3 Ea]) that holds each reference column"""
    Ea = 64 * head_slots(d * H, H) * H
    cols = slot_columns(d, H)
    return torch.cat([s * Ea + cols for s in range(3)])


def rope_pair_sum(t: torch.Tensor, E: int, H: int) -> torch.Tensor:
    """t [M, >= 2E] in the reference's column order: both members of every rotate-half pair (j, j + d/2) of the q and
    k heads replaced by their sum (the bound of a rotation by |cos|, |sin| <= 1 of two bounded values)"""
    d = E // H
    t = t.clone()
    qk = t[:, :2 * E].view(-1, 2, H, 2, d // 2)
    qk[:] = qk.sum(3, keepdim=True)
    return t


def qkv_ref_heads(a, w, bias, q_scale, H, T=None, cos=None, sin=None):
    """[q*scale | k | v] in float64 in the reference's layout (w [3E, K] and bias [3E] in the reference's row order,
    unpadded), the bias added before the scale, with rotary_embedding.py's rotate-half on every q and k head of width
    d = E / H: (x1, x2) = the head's halves, (x1 cos - x2 sin, x2 cos + x1 sin) under the [T, d/2] table (row r at
    position r % T).  Returns (y, absdot) with absdot the matching sum of |products| (rotated pairs: both members'
    sums).  At d = 64 this is qkv_ref."""
    y, absdot = gemm_exact(a, w, bias)
    E = y.shape[1] // 3
    d = E // H
    y[:, :E] *= q_scale
    absdot[:, :E] *= q_scale
    if cos is not None:
        M = y.shape[0]
        t = torch.arange(M, device=y.device) % T
        c, s = cos.double()[t][:, None, None, :d // 2], sin.double()[t][:, None, None, :d // 2]
        qk = y[:, :2 * E].view(M, 2, H, d)
        x1, x2 = qk[..., :d // 2].clone(), qk[..., d // 2:].clone()
        qk[..., :d // 2], qk[..., d // 2:] = x1 * c - x2 * s, x2 * c + x1 * s
        absdot = rope_pair_sum(absdot, E, H)
    return y, absdot


def qkv_bound(y: torch.Tensor, absdot: torch.Tensor, K: int) -> torch.Tensor:
    """|out - y| of the fp16 QKV epilogue: gemm_acc_bound, the q scale and the rotation's products and add (4 u |y|),
    and the fp16 output"""
    return gemm_acc_bound(absdot, K, y) + 4 * U32 * y.abs() + f16_bound(y)


# ---- GEMM launch table ----------------------------------------------------------------------------------------------
# (name, layers, embed_dim, heads, ffn_dim, rotary, msa)
MODELS: Dict[str, Tuple[int, int, int, int, bool, bool]] = {
    "esm2_t6_8M": (6, 320, 20, 1280, True, False),
    "esm2_t12_35M": (12, 480, 20, 1920, True, False),
    "esm2_t30_150M": (30, 640, 20, 2560, True, False),
    "esm2_t33_650M": (33, 1280, 20, 5120, True, False),
    "esm2_t36_3B": (36, 2560, 40, 10240, True, False),
    "esm2_t48_15B": (48, 5120, 40, 20480, True, False),
    "esm1b_t33_650M": (33, 1280, 20, 5120, False, False),
    "esm_msa1b_t12_100M": (12, 768, 12, 3072, False, True),
}
VOCAB = 33


def head_slots(E: int, H: int) -> int:
    """64-wide column slots per head on the attention side (api.cu head_slots)."""
    return 2 if E // H > 64 else 1


def gemm_launches(name: str) -> List[Tuple[str, int, int, int]]:
    """[(role, epilogue, N, K)] of one forward of the model: the transformer layer's four GEMMs (the MSA layer has a
    row and a column attention block, each with its QKV and out-projection), then the LM head's dense layer
    (erf-GELU into fp32) and its projection onto the vocabulary padded to 64 columns."""
    _, E, H, F, _, msa = MODELS[name]
    Ea = 64 * head_slots(E, H) * H
    attn = [("qkv", EPI_QKV_ROPE, 3 * Ea, E), ("out_proj", EPI_BIAS_RESIDUAL, E, Ea)]
    ffn = [("fc1", EPI_BIAS_GELU, F, E), ("fc2", EPI_BIAS_RESIDUAL, E, F)]
    layer = (attn + attn if msa else attn) + ffn
    npad = (VOCAB + 63) // 64 * 64
    return layer + [("lm_dense", EPI_BIAS_GELU_F32, E, E), ("lm_out", EPI_BIAS_F32, npad, E)]


def fp32x3_accepts(E: int, H: int) -> bool:
    """The layers run precision 1 (fp32x3) when E % 64 == 0 (every GEMM K a whole number of 64-wide slabs) and the
    heads fit one 64-wide slot (model.py ProteinLanguageModel.set_precision; the MSA layers have head_dim 64)."""
    return E % 64 == 0 and E // H <= 64


# 8M, 150M, 650M, 3B, ESM-1b and MSA-1b; 35M fails E % 64 (480) and 15B has 128-wide heads
FP32X3_MODELS: List[str] = [n for n, (_, E, H, _, _, _) in MODELS.items() if fp32x3_accepts(E, H)]


def packed_bytes_from_launches(name: str) -> int:
    """esmb200_layer_packed_bytes of the model's transformer layer, from the B operands [N, K] fp16 of its four
    GEMMs, each 1024-byte aligned (api.cu packed_layout)."""
    launches = gemm_launches(name)[:4]
    return sum((n * k * 2 + 1023) // 1024 * 1024 for _, _, n, k in launches)


# ---- fp32x3 operands ------------------------------------------------------------------------------------------------
F16_HALF_QUANTUM = 2.0 ** -25  # half the smallest fp16 subnormal (2^-24): the absolute rounding error below 2^-14


def split16(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """fp32 x -> fp16 (hi, lo) with hi = rn16(x), lo = rn16(x - hi) (esmb200_convert_split; the GEMM epilogues and the
    attention kernels split their fp32 results the same way).  x - hi is exact in fp32."""
    x = x.float()
    hi = x.half()
    return hi, (x - hi.float()).half()


def join64(hi: torch.Tensor, lo: torch.Tensor) -> torch.Tensor:
    """The value a hi | lo pair stands for, in float64 (exact)."""
    return hi.double() + lo.double()


def split_rep_bound(x: torch.Tensor) -> torch.Tensor:
    """|x - (hi + lo)| for (hi, lo) = split16(x): r = x - hi is exact and |r| <= 2^-11 |x| (or <= 2^-25 when hi is
    subnormal); rn16(r) is within 2^-11 |r| + 2^-25 of r, the 2^-25 being the subnormal half-quantum, which applies to
    the lo half of every |x| below ~2^-3.  Hence <= 2^-22 |x| + 2^-25."""
    return 2.0 ** -22 * x.double().abs() + F16_HALF_QUANTUM


def split_acc_bound(a_hi: torch.Tensor, a_lo: torch.Tensor, w_hi: torch.Tensor, w_lo: torch.Tensor, K: int,
                    y: torch.Tensor) -> torch.Tensor:
    """|out - y| for the split GEMM (gemm2_f16_kernel<EPI, true>) before any epilogue function, y = (a_hi + a_lo)
    (w_hi + w_lo)^T + bias in float64 (a [M, K], w [N, K] fp16 halves):
      * the three passes hi*hi, lo*hi, hi*lo feed one fp32 accumulator, 3K/16 k16 steps; each step adds its exact
        products with truncation (one ulp, 2^-23 of a partial sum bounded by the absolute sum of all three passes),
        doubled for slack and given 4 steps of headroom as for the fp16 kernel: (3K/16 + 4) 2^-22 sum|a w|;
      * the dropped lo*lo term, bounded by sum_k |a_lo w_lo| (computed exactly, <= 2^-22 sum|a w|);
      * the bias add and the fp32 result: 2 u |y|."""
    ah, al, wh, wl = (t.double().abs() for t in (a_hi, a_lo, w_hi, w_lo))
    passes = ah @ wh.t() + al @ wh.t() + ah @ wl.t()
    return (3 * K / 16 + 4) * 2.0 ** -22 * passes + al @ wl.t() + 2 * U32 * y.abs()


def split_box_scale(K: int) -> float:
    """(3K/16 + 4) 2^-25: the scale of the per-output-box rel-Frobenius gate of the split GEMM (the accumulation drift
    of DESIGN.md section 4, per unit of relative size)."""
    return (3 * K / 16 + 4) * 2.0 ** -25


# ---- fp16 attention -------------------------------------------------------------------------------------------------
# The fp16 attention kernels, per key block of `block` keys (128: attention_wg_kernel, 64: attention_fwd_kernel<false,
# 2>): S = q k^T on the tensor cores (fp32, truncating k16 steps over the head's D = 64 or 128 columns, both slots into
# one accumulator); the exact running maximum m; e = ex2.approx(fma(s, log2e, -m log2e)) in fp32; l = alpha l + sum e
# (fp32); O = alpha O + fp16(e) V (fp32, truncating k16 steps); ctx = fp16(O * (1 / l)).  alpha = ex2.approx((m_old - m)
# log2e) multiplies O and l alike, so its own error cancels in ctx.  The probability kernel recomputes S (mma.sync,
# another accumulation order than the wgmma forward) and writes ex2.approx(fma(s, log2e, -m log2e)) * (1 / l) with the
# forward's saved m and l.
F16_U = 2.0 ** -11  # unit roundoff of fp16


def attention64(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, padded: Optional[torch.Tensor], block: int) -> Dict:
    """float64 softmax attention of fp16 queries q [B, H, Tq, D] on keys and values k, v [B, H, T, D] (D = 64 or 128)
    under the key-padding mask `padded` [B, T] (True: padded key; None: none), with what the error bounds below need.
    q may be any slice of a head's query rows (attention64_rows): every row's values depend on that row and the keys
    alone.  Rows of an all-padding sequence are 0 (ctx, p, m and l).
      * lerr [B,H,Tq,T]: the absolute error bound of each logit, (D/16 + 4) 2^-22 sum_d |q_d k_d| (the GEMM's
        accumulation bound: D/16 truncating k16 steps, one ulp of a partial sum bounded by sum|q k| each, doubled,
        plus 4 steps);
      * delta [B,H,Tq,T]: the relative error bound Delta_j of key j's unnormalised weight e^(s_j - m): its logit
        (lerr), ex2.approx (2 ulp = 2^-22, doubled) and the fp32 roundings of log2e, s log2e and -m log2e
        (2^-23 (|s| + 3 |m|));
      * nblk [B,1,1,1]: the key blocks the kernel walks, ceil(kvlen / block), kvlen = 1 + the last attendable key."""
    q, k, v = q.double(), k.double(), v.double()
    B, H, T, D = k.shape
    if padded is None:
        padded = torch.zeros(B, T, dtype=torch.bool, device=q.device)
    padded = padded.bool()
    km = padded[:, None, None, :]
    s = q @ k.transpose(-1, -2)
    sm = s.masked_fill(km, float("-inf"))
    m = sm.amax(-1, keepdim=True)
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    e = torch.exp(sm - m)
    l = e.sum(-1, keepdim=True)
    p = e / torch.where(l > 0, l, torch.ones_like(l))
    lerr = ((D / 16 + 4) * 2.0 ** -22 * (q.abs() @ k.abs().transpose(-1, -2))).masked_fill(km, 0.0)
    delta = (lerr + 2.0 ** -21 + 2.0 ** -23 * (s.abs() + 3 * m.abs())).masked_fill(km, 0.0)
    idx = torch.arange(1, T + 1, device=q.device)
    kvlen = torch.where(padded, torch.zeros_like(idx), idx).amax(-1)
    nblk = ((kvlen + block - 1) // block).double()[:, None, None, None]
    return dict(q=q, k=k, v=v, s=s, m=m, l=l, p=p, ctx=p @ v, lerr=lerr, delta=delta, nblk=nblk, km=km, block=block)


def attention64_rows(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, padded: Optional[torch.Tensor], block: int,
                     max_elems: int = 1 << 23):
    """attention64 over consecutive slices of the query rows, so that one head at T = 16384 fits a few GB: yields
    (i0, r), r = attention64(q[..., i0:i0 + n, :], k, v, padded, block), with n rows per slice (the last may have
    fewer) such that a [B, H, n, T] tensor holds at most max_elems elements (at least one row).  The element-wise
    values and bounds of a slice are those of the same rows of the whole-head reference; the per-head gate is
    attn_relfro_combine of the slices' attn_relfro_terms, summed."""
    B, H, Tq, _ = q.shape
    n = max(1, max_elems // (B * H * k.shape[-2]))
    for i0 in range(0, Tq, n):
        yield i0, attention64(q[..., i0:i0 + n, :], k, v, padded, block)


def _vsum(r, f) -> torch.Tensor:
    """[B,H,1,D]: sum over the attendable keys of f(v)"""
    return f(r["v"]).masked_fill(r["km"].transpose(-1, -2), 0.0).sum(-2, keepdim=True)


def _safe(l: torch.Tensor) -> torch.Tensor:
    return torch.where(l > 0, l, torch.ones_like(l))


def attn_weights(r) -> torch.Tensor:
    """The weights' share of the ctx bound, element-wise: ctx moves by sum_j p_j Delta_j (v_j - ctx), at most
    (p Delta) |v| + (sum_j p_j Delta_j) |ctx|."""
    pd = r["p"] * r["delta"]
    return pd @ r["v"].abs() + pd.sum(-1, keepdim=True) * r["ctx"].abs()


def attn_acc(r) -> torch.Tensor:
    """The accumulations' share of the ctx bound, element-wise:
      * P . V: nblk block/16 truncating k16 steps into one fp32 accumulator, each within 2^-22 of a partial sum bounded
        by sum_j P_j |v_j| (P = fp16(e) <= (1 + 2^-11) e), plus 4 steps, as for the GEMM; and the rescale of O once per
        block (u each);
      * the row sum: at most 10 fp32 roundings per block on any path of l (the pair sum, up to 8 running adds, the
        rescale), the quad shuffle sum (2), 1 / l and O * (1 / l): (10 nblk + 8) u relative."""
    nblk = r["nblk"]
    pv = r["p"] @ r["v"].abs()
    b = ((nblk * r["block"] / 16 + 4) * 2.0 ** -22 * (1 + F16_U) + nblk * U32) * pv
    return b + (10 * nblk + 8) * U32 * r["ctx"].abs()


def attn_ctx_bound(r) -> torch.Tensor:
    """|ctx - ctx64| element-wise: attn_weights, attn_acc, P rounded to fp16 relative to the running maximum (2^-11 e_j,
    or the subnormal half-quantum 2^-25 below 2^-14, per key: 2^-11 p |v| + 2^-25 sum_j |v_j| / l after normalisation,
    the rescales only shrinking it; not normalised away, since l sums the fp32 e, not fp16(e)), and the fp16 output
    (2^-11 |ctx| + 2^-25)."""
    p, v, ctx, l = r["p"], r["v"], r["ctx"], r["l"]
    b = attn_weights(r) + attn_acc(r) + F16_U * (p @ v.abs()) + F16_HALF_QUANTUM * _vsum(r, torch.abs) / _safe(l)
    return b + F16_U * ctx.abs() + F16_HALF_QUANTUM


def half_ulp16(y: torch.Tensor) -> torch.Tensor:
    """half an fp16 ulp at |y| (2^-25 in the subnormal range)"""
    _, ex = torch.frexp(y.double().abs())
    return torch.ldexp(torch.ones_like(y, dtype=torch.float64), (ex - 1).clamp_min(-14) - 11)  # exact, unlike pow


GATE_SIGMAS = 3.0


def attn_relfro_gate(r) -> torch.Tensor:
    """[B, H]: the per-(sequence, head) bound of ||ctx - ctx64||_F / ||ctx64||_F over r's query rows,
    attn_relfro_combine(*attn_relfro_terms(r)).
    The errors that do not depend on the sign of v are modelled as independent and zero-mean:
      * the fp16 roundings of P and of the output, uniform within half an ulp (variance ulp^2 / 12): P's half ulp taken
        at its upper bound 2^-11 e_j (2^-25 below 2^-14), the output's as the exact half ulp of ctx64;
      * each weight's error, at most Delta_j in size with a sign set by q and k alone (the logit's accumulation,
        ex2.approx, the exponent's roundings), so independent of v_j's: variance p_j^2 Delta_j^2 (|v_j| + |ctx|)^2.
    The squared error norm sums at least 64 T such terms, so it concentrates within a few per cent of its mean sigma^2;
    GATE_SIGMAS = 3 sigma covers what the model approximates (errors that are not quite uniform or independent).  The
    accumulations truncate, a bias rather than noise: attn_acc is added at its worst case.
    Diffuse heads give a gate of ~1.3e-3 (P and the output each ~2^-11 / sqrt(3) relative); ctx scaled by 1 + 2^-9
    (1.95e-3) is outside it."""
    return attn_relfro_combine(*attn_relfro_terms(r))


def attn_relfro_terms(r) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """([B, H] each) the sums over r's query rows and head dimensions of the gate's variance sigma^2 (the model of
    attn_relfro_gate), of attn_acc^2 and of ctx64^2.  Sums over the row slices of a head give the whole head's."""
    p, v, ctx, l = r["p"], r["v"], r["ctx"], r["l"]
    var = (F16_U ** 2 / 3) * ((p * p) @ (v * v)) + (F16_HALF_QUANTUM ** 2 / 3) * _vsum(r, torch.square) / _safe(l) ** 2
    var = var + half_ulp16(ctx) ** 2 / 3
    w2 = (p * r["delta"]).pow(2)
    var = var + w2 @ (v * v) + 2 * (w2 @ v.abs()) * ctx.abs() + w2.sum(-1, keepdim=True) * ctx * ctx
    return var.sum((-1, -2)), attn_acc(r).pow(2).sum((-1, -2)), ctx.pow(2).sum((-1, -2))


def attn_relfro_combine(var: torch.Tensor, acc2: torch.Tensor, ctx2: torch.Tensor) -> torch.Tensor:
    """the gate (GATE_SIGMAS sigma + ||attn_acc||_F) / ||ctx64||_F from the sums of attn_relfro_terms"""
    return (GATE_SIGMAS * var.sqrt() + acc2.sqrt()) / ctx2.sqrt().clamp_min(1e-300)


def attn_probs_bound(r) -> torch.Tensor:
    """|p - p64| of the probability kernel: p_j off by Delta_j (its own, recomputed logit, ex2.approx and argument
    roundings), the saved row sum off by sum_i p_i Delta_i <= max Delta (the forward's logits) plus the roundings of
    its rescale chain: the exponents (m_old - m) log2e, 3 u sum |m_old - m| <= 3 u (|m| + |m_first|) <= max Delta (Delta
    of the first block's maximum alone holds 34 u |m_first| + 6 u |m|), and ex2.approx of alpha (8 u per block); the row
    sum's own (10 nblk + 8) u, 1 / l, the product and the fp32 store (4 u).  ex2.approx flushes results below 2^-126 to
    zero.  The saved maximum's error cancels: it enters the forward's l and the probability alike."""
    p, delta, nblk = r["p"], r["delta"], r["nblk"]
    dmax = delta.amax(-1, keepdim=True)
    return p * (delta + 2 * dmax + (18 * nblk + 12) * U32) + 2.0 ** -126


def attn_rowsum_bound(r) -> torch.Tensor:
    """[B,H,T]: |sum_j p_j - 1| of the probability kernel's rows.  Row j's numerator and the saved row sum carry the
    same weights, each off by its own Delta (the probability kernel's recomputed logit and the forward's), so the
    weight errors cost sum_j p_j (Delta'_j + Delta_j) <= 2 sum_j p_j Delta_j rather than max Delta; what the row sum
    alone carries is its rescale chain, the exponents 3 u sum |m_old - m| <= 6 u max|s| over the valid keys and
    ex2.approx of alpha (8 u per block), its own (10 nblk + 8) u, and 1 / l, the product and the fp32 stores (4 u).
    Unlike the sum of the element bounds this is tighter than a common rescale of the row: on diffuse heads
    p (1 + 2^-13) leaves it."""
    p, delta, nblk = r["p"], r["delta"], r["nblk"][..., 0]
    smax = r["s"].abs().masked_fill(r["km"], 0.0).amax(-1)
    return 2 * (p * delta).sum(-1) + 6 * U32 * smax + (18 * nblk + 12) * U32


def attn_max_bound(r) -> torch.Tensor:
    """[B,H,T]: |saved row max - m64|: the saved maximum is the largest of the kernel's own fp32 logits, so within the
    row's largest logit error"""
    return r["lerr"].amax(-1) + 1e-30


def attn_sum_bound(r, l_at: torch.Tensor) -> torch.Tensor:
    """[B,H,T]: |saved row sum - l_at|, l_at = sum_j e^(s_j - m_saved) in float64: the weights' Delta (<= max Delta),
    the rescale chain's exponents (<= max Delta, see attn_probs_bound) and ex2.approx (8 u per block), and the sum's
    (10 nblk + 8) u"""
    dmax = r["delta"].amax(-1)
    return l_at * (2 * dmax + (18 * r["nblk"][..., 0] + 8) * U32) + 1e-30


# ---- tied row attention (MSA Transformer) ---------------------------------------------------------------------------
# csrc/tied_attention.cuh, <false> (fp16) and <true> (fp32x3): tied_scores_kernel S = sum_r q_r k_r^T on the tensor
# cores (fp16: one fp32 accumulator carried over all R alignment rows, 4 truncating k16 steps per row; fp32x3: each
# row's 64-wide slab in a fresh fragment, 3 passes q_lo k_hi, q_hi k_lo, q_hi k_hi per k16 step, then one fp32 add into
# the running sum); tied_softmax_kernel, one warp per row: -10000 at padded key columns, the exact row max m,
# e = __expf(x - m) (ex2.approx of fp32 (x - m) log2e), a row sum of ceil(C/32) serial terms per lane then 5 shuffle
# levels, q = e * (1.0f / sum) (a correctly rounded divide: no --use_fast_math), P = fp16(q) or hi | lo of q, zero in
# columns [C, Cp); tied_pv_kernel ctx = P V over Cp/16 truncating k16 steps (fp32x3: P_hi v_hi, P_lo v_hi, P_hi v_lo per
# step), fp16 or hi | lo output.
def tied_operands(qkv: torch.Tensor, B: int, R: int, C: int, H: int, split: bool):
    """The kernel's operands in float64, [B,R,C,3,H,64] (sections q, k, v): (value, hi, lo); fp16: (x, x, None)."""
    y = qkv.double().view(B, R, C, 6 if split else 3, H, 64)
    if split:
        return y[:, :, :, :3] + y[:, :, :, 3:], y[:, :, :, :3], y[:, :, :, 3:]
    return y, y, None


def _qk(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    return torch.einsum("brihd,brjhd->hbij", a, b)


def _pv(p: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    return torch.einsum("hbij,brjhd->brihd", p, v)


def tied_depth(C: int) -> int:
    """rounding depth of tied_softmax_kernel's row sum: ceil(C/32) - 1 serial adds per lane, then 5 shuffle levels"""
    return (C + 31) // 32 + 4


def tied_pad(key_pad: Optional[torch.Tensor], B: int, C: int, device) -> torch.Tensor:
    """[1,B,1,C] bool: padded key columns (key_pad [B,C], 1 = padded; None: none)"""
    if key_pad is None:
        return torch.zeros(1, B, 1, C, dtype=torch.bool, device=device)
    return key_pad.bool().view(1, B, 1, C)


def tied64(qkv: torch.Tensor, key_pad: Optional[torch.Tensor], B: int, R: int, C: int, H: int, split: bool) -> Dict:
    """float64 tied row attention on the kernel's own operands (qkv [B*R*C, 3E] fp16, or [B*R*C, 6E] hi | lo):
    S = sum_r q_r k_r^T [H,B,C,C], -10000 at padded key columns, P = softmax, ctx = P v_r [B,R,C,H,64]; and lerr, the
    bound of each of the kernel's fp32 logits:
      * fp16: 4R truncating k16 steps into one accumulator, (4R + 4) 2^-22 sum|q k| (attention64's lerr, D = 64 R);
      * fp32x3: per alignment row a fresh fragment of 12 steps, (12 + 4) 2^-22 times the slab's
        sum(|q_hi k_hi| + |q_lo k_hi| + |q_hi k_lo|), the dropped sum|q_lo k_lo|, and the R fp32 adds of the slabs into
        the running sum, sum_bound over the slabs' absolute sums (each within 2^-10 of sum|q k|)."""
    x, hi, lo = tied_operands(qkv, B, R, C, H, split)
    q, k, v = x[:, :, :, 0], x[:, :, :, 1], x[:, :, :, 2]
    s = _qk(q, k)
    qk_abs = _qk(q.abs(), k.abs())
    if split:
        qh, kh, ql, kl = hi[:, :, :, 0].abs(), hi[:, :, :, 1].abs(), lo[:, :, :, 0].abs(), lo[:, :, :, 1].abs()
        passes = _qk(qh, kh) + _qk(ql, kh) + _qk(qh, kl)
        lerr = 16 * 2.0 ** -22 * passes + _qk(ql, kl) + sum_bound(qk_abs * (1 + 2.0 ** -10), R)
    else:
        lerr = (4 * R + 4) * 2.0 ** -22 * qk_abs
    km = tied_pad(key_pad, B, C, qkv.device)
    sm = s.masked_fill(km, -10000.0)
    m = sm.amax(-1, keepdim=True)
    p = torch.softmax(sm, -1)
    return dict(s=s, sm=sm, m=m, p=p, v=v, ctx=_pv(p, v), lerr=lerr, km=km, split=split, R=R, C=C,
                Cp=(C + 63) // 64 * 64)


def tied_softmax64(S: torch.Tensor, key_pad: Optional[torch.Tensor]) -> Dict:
    """float64 softmax of the kernel's own fp32 logits S [H,B,C,C] (-10000 at padded key columns), with Delta_j, the
    relative error bound of the kernel's e_j = __expf(x_j - m): the fp32 roundings of x - m, of the product with log2e
    and of log2e itself (3 u |x - m|), and ex2.approx (2^-22, doubled)."""
    H, B, C, _ = S.shape
    x = S.double().masked_fill(tied_pad(key_pad, B, C, S.device), -10000.0)
    m = x.amax(-1, keepdim=True)
    return dict(p=torch.softmax(x, -1), delta=3 * U32 * (x - m).abs() + 2.0 ** -21, C=C)


def tied_probs_bound(sr: Dict) -> torch.Tensor:
    """|q - p| for the kernel's fp32 q = e_j * (1 / sum) (the attn_probs output) against p = softmax(S_kernel): its own
    weight's Delta_j, the row sum's weights sum_i p_i Delta_i, the sum's tied_depth(C) roundings, 1 / sum and the
    product (u each); results of ex2.approx below 2^-126 may be subnormal or flushed to zero (2^-126 absolute)."""
    p, d = sr["p"], sr["delta"]
    return p * (d + (p * d).sum(-1, keepdim=True) + (tied_depth(sr["C"]) + 2) * U32) + 2.0 ** -126


def tied_P_bound(sr: Dict, split: bool) -> torch.Tensor:
    """|P - p| for the kernel's P: tied_probs_bound, then fp16(q) (half an ulp, at most 2^-11 |q| or the subnormal
    half-quantum 2^-25) or the hi | lo pair of q (split_rep_bound)."""
    b = tied_probs_bound(sr)
    q = sr["p"] + b
    return b + (split_rep_bound(q) if split else F16_U * q + F16_HALF_QUANTUM)


def tied_rowsum_bound(C: int) -> float:
    """|sum_j q_j - 1| for a row of the fp32 probabilities.  Every q_j is e_j (1 + e_mul) / (sum_i e_i (1 + e_sum)) with
    the kernel's own e_i in numerator and sum alike, so the weights' errors cancel: what is left is the sum's tied_depth(C)
    roundings, 1 / sum and the product (u each), and C flushed terms below 2^-126.  A uniform rescale of the row by
    1 + 2^-13 is ~30 times outside it at C = 1024."""
    return (tied_depth(C) + 2) * U32 + C * 2.0 ** -126


def tied_pv(P_hi: torch.Tensor, P_lo: Optional[torch.Tensor], v_hi: torch.Tensor, v_lo: Optional[torch.Tensor],
            Cp: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """float64 P V on the kernel's own P ([H,B,C,C] halves, the columns [C, Cp) being zero) and v ([B,R,C,H,64] halves)
    -> (ctx [B,R,C,H,64], bound of the kernel's ctx):
      * fp16: Cp/16 truncating k16 steps, (Cp/16 + 4) 2^-22 sum_j P_j |v_j|, and half an fp16 ulp of the output;
      * fp32x3: three passes, (3 Cp/16 + 4) 2^-22 sum_j (|P_hi v_hi| + |P_lo v_hi| + |P_hi v_lo|), the dropped
        sum_j |P_lo v_lo|, and the hi | lo output (split_rep_bound)."""
    if P_lo is None:
        ref = _pv(P_hi, v_hi)
        acc = (Cp / 16 + 4) * 2.0 ** -22 * _pv(P_hi.abs(), v_hi.abs())
        return ref, acc + half_ulp16(ref.abs() + acc)
    ph, pl, vh, vl = P_hi.abs(), P_lo.abs(), v_hi.abs(), v_lo.abs()
    ref = _pv(P_hi + P_lo, v_hi + v_lo)
    acc = (3 * Cp / 16 + 4) * 2.0 ** -22 * (_pv(ph, vh) + _pv(pl, vh) + _pv(ph, vl)) + _pv(pl, vl)
    return ref, acc + split_rep_bound(ref.abs() + acc)


def _tied_delta(r: Dict) -> torch.Tensor:
    """relative error bound of each weight e_j: its logit (lerr; none at a padded column, whose logit is replaced) and
    the softmax's own Delta_j"""
    return r["lerr"].masked_fill(r["km"], 0.0) + 3 * U32 * (r["sm"] - r["m"]).abs() + 2.0 ** -21


def _tied_acc(r: Dict) -> torch.Tensor:
    """the accumulations' worst case, element-wise: P V (tied_pv's accumulation, on P within 2^-10 of p; fp32x3 also
    its dropped lo*lo), and the row sum, 1 / sum and the product (tied_depth(C) + 2) u of sum_j p_j |v_j|"""
    pv = _pv(r["p"], r["v"].abs())
    steps = (3 if r["split"] else 1) * r["Cp"] / 16 + 4
    rel = steps * 2.0 ** -22 * (1 + 2.0 ** -10) + (tied_depth(r["C"]) + 2) * U32
    if r["split"]:
        rel = rel + 2.0 ** -22
    return rel * pv


def tied_ctx_bound(r: Dict) -> torch.Tensor:
    """|ctx - ctx64| element-wise ([B,R,C,H,64]) from tied64, in attn_ctx_bound's structure: the weights' errors
    sum_j p_j Delta_j (v_j - ctx) (Delta_j the logit bound plus the softmax's), _tied_acc, P's representation (fp16:
    2^-11 p_j or 2^-25 per key; fp32x3: 2^-22 p_j + 2^-25) and the output's (fp16: 2^-11 |ctx| + 2^-25; fp32x3:
    split_rep_bound).  Loose for fp16 at large R, where the logit bound grows as R^1.5."""
    p, v, ctx = r["p"], r["v"], r["ctx"]
    pd = p * _tied_delta(r)
    va = v.abs()
    b = _pv(pd, va) + pd.sum(-1).permute(1, 2, 0)[:, None, :, :, None] * ctx.abs() + _tied_acc(r)
    vsum = va.sum(2, keepdim=True)  # [B,R,1,H,64]: sum over the keys of |v_j|
    rep = (2.0 ** -22 if r["split"] else F16_U) * _pv(p, va) + F16_HALF_QUANTUM * vsum
    out = split_rep_bound(ctx) if r["split"] else F16_U * ctx.abs() + F16_HALF_QUANTUM
    return b + rep + out


def tied_relfro_gate(r: Dict) -> torch.Tensor:
    """[B, H]: the per-(alignment, head) bound of ||ctx - ctx64||_F / ||ctx64||_F over the alignment's R x C x 64
    outputs, in attn_relfro_gate's model: P's and the output's roundings uniform and independent (variance ulp^2 / 12
    at their upper bounds), each weight's error at most Delta_j with a sign independent of v_j, GATE_SIGMAS sigma of
    that, plus _tied_acc at its worst case."""
    p, v, ctx = r["p"], r["v"], r["ctx"]
    rel = 2.0 ** -22 if r["split"] else F16_U
    var = (rel ** 2 / 3) * _pv(p * p, v * v) + (F16_HALF_QUANTUM ** 2 / 3) * (v * v).sum(2, keepdim=True)
    var = var + (split_rep_bound(ctx) if r["split"] else half_ulp16(ctx)) ** 2 / 3
    w2 = (p * _tied_delta(r)).pow(2)
    w2sum = w2.sum(-1).permute(1, 2, 0)[:, None, :, :, None]
    var = var + _pv(w2, v * v) + 2 * _pv(w2, v.abs()) * ctx.abs() + w2sum * ctx * ctx
    sigma = var.sum((1, 2, 4)).sqrt()
    acc = _tied_acc(r).pow(2).sum((1, 2, 4)).sqrt()
    return (GATE_SIGMAS * sigma + acc) / ctx.pow(2).sum((1, 2, 4)).sqrt().clamp_min(1e-300)


# ---- erf-GELU -------------------------------------------------------------------------------------------------------
AS_ERF = 1.5e-7  # Abramowitz & Stegun 7.1.26: |erf(z) - approx| <= 1.5e-7 for z >= 0


def gelu64(x: torch.Tensor) -> torch.Tensor:
    x = x.double()
    return x * 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_bound(x: torch.Tensor) -> torch.Tensor:
    """|gelu_erf(x) - gelu(x)| bound for the fp32 epilogue, x the fp32 pre-activation (float64 tensor).
    gelu_erf computes q = 0.5 erfc(|x|/sqrt2) as 0.5 poly(t) exp(-z^2) and returns x (1 - q) or x q:
      * the A&S truncation: |dq| <= 0.5 * 1.5e-7;
      * rcp.approx (t, 1 ulp), the four fmas of the Horner chain, ex2.approx (2 ulp) and the rounding of its argument
        -z^2 log2(e) (|arg| ulp, times ln 2) perturb q relatively by at most 32 u + 2 u |arg|, with the Horner
        chain's condition number (|t P'(t) / P(t)| <= 3.5 on t in (0, 1], P = t (a1 + a2 t + ...)) folded in;
      * the final 1 - q and x * (...) roundings: 2 u |y|.
    Tightening any term below what the kernel computes makes the test fail on a correct kernel."""
    x = x.double()
    z = x.abs() / math.sqrt(2.0)
    q = 0.5 * torch.erfc(z)
    arg = z * z / math.log(2.0)
    return x.abs() * (0.5 * AS_ERF + q * (32 + 2 * arg) * U32) + 2 * U32 * gelu64(x).abs() + 1e-30


def horner_condition() -> float:
    """max over t in (0, 1] of |t P'(t) / P(t)| for the A&S polynomial P (the factor folded into gelu_bound)."""
    a = [0.254829592, -0.284496736, 1.421413741, -1.453152027, 1.061405429]
    t = torch.linspace(1e-6, 1.0, 100001, dtype=torch.float64)
    p = sum(c * t ** (i + 1) for i, c in enumerate(a))
    dp = sum((i + 1) * c * t ** i for i, c in enumerate(a))
    return float((t * dp / p).abs().max())


# ---- LayerNorm ------------------------------------------------------------------------------------------------------
def layer_norm64(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    return torch.nn.functional.layer_norm(x.double(), (x.shape[-1],), w.double(), b.double(), eps)


def ln_tol(E: int, cond: float = 1.0) -> float:
    """Bound of an fp32 two-pass LayerNorm row, relative to ln_scale: the mean and variance of E fp32 values (a rounding
    walk of ~sqrt(E) steps, so |d mean| / std <~ sqrt(E) u cond with cond = |mean| / std of the row), rsqrt (2 ulp) and
    the affine step (3 roundings), with a factor 4 of room (the bound of tests/test_gpu_row_kernels.py)."""
    return 4 * U32 * (8 + 2 * E ** 0.5 * (1 + cond))


def ln_scale(want: torch.Tensor, w: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """|g| (|xhat| + 1) + |b| for want = g xhat + b: what ln_tol is relative to"""
    return (want - b.double()).abs() + w.double().abs() + b.double().abs()


# ---- embedding prologues --------------------------------------------------------------------------------------------
KEEP_SCALE = 1 - 0.15 * 0.8  # esm2.py:90: the share of tokens the training-time dropout left in place


def positions(tokens: torch.Tensor, padding_idx: int) -> torch.Tensor:
    """LearnedPositionalEmbedding.forward (esm/modules.py:247-248) over the last dim: the count of non-pad tokens up to
    and including this one, plus padding_idx; padding_idx at the pads themselves."""
    nonpad = tokens.ne(padding_idx).long()
    return torch.cumsum(nonpad, -1) * nonpad + padding_idx


def mask_ratio(tokens: torch.Tensor, padding_idx: int, mask_idx: int) -> torch.Tensor:
    """[B] float64: n_mask / n_nonpad (0 / 0 = NaN for a sequence of pads only)"""
    return tokens.eq(mask_idx).sum(-1).double() / tokens.ne(padding_idx).sum(-1).double()


def embed_esm2_64(tokens: torch.Tensor, table: torch.Tensor, padding_idx: int, mask_idx: int,
                  token_dropout: bool) -> torch.Tensor:
    """esm/model/esm2.py:84-95 in float64: gather, <mask> rows zeroed and (x 0.88) / (1 - n_mask / n_nonpad) only under
    token_dropout, pad rows multiplied by zero (so a NaN scale stays NaN there, as in the reference).
    tokens [B,T] -> [B,T,E]."""
    x = table.double()[tokens]
    if token_dropout:
        x = x.masked_fill(tokens.eq(mask_idx)[..., None], 0.0)
        x = x * KEEP_SCALE / (1 - mask_ratio(tokens, padding_idx, mask_idx))[:, None, None]
    return x * tokens.ne(padding_idx)[..., None].double()


def embed_scale_bound(tokens: torch.Tensor, padding_idx: int, mask_idx: int, token_dropout: bool) -> torch.Tensor:
    """[B,1,1]: the relative error of the fp32 token-dropout scale. 0.88 as an fp32 constant, the product and the
    quotient are one rounding each; the ratio r and 1 - r are one each, and the ratio's reaches 1 - r magnified by
    r / (1 - r): u (4 + r / (1 - r)).  Without token_dropout the gather is exact."""
    if not token_dropout:
        return torch.zeros(tokens.shape[0], 1, 1, dtype=torch.float64)
    r = mask_ratio(tokens, padding_idx, mask_idx).cpu()
    return (U32 * (4 + r / (1 - r)))[:, None, None].nan_to_num(nan=0.0, posinf=0.0)


def embed_esm1b_64(tokens, table, pos_table, ln_w, ln_b, padding_idx: int, mask_idx: int, token_dropout: bool,
                   eps: float = 1e-5):
    """esm/model/esm1.py:121-139 in float64: the ESM-2 scaling of the token embedding, plus the learned position, then
    emb_layer_norm_before when ln_w is given, then pad rows multiplied by zero.  Returns (x, the rows before the
    LayerNorm and the pad zeroing)."""
    x = table.double()[tokens]
    if token_dropout:
        x = x.masked_fill(tokens.eq(mask_idx)[..., None], 0.0)
        x = x * KEEP_SCALE / (1 - mask_ratio(tokens, padding_idx, mask_idx))[:, None, None]
    pre = x + pos_table.double()[positions(tokens, padding_idx)]
    x = layer_norm64(pre, ln_w, ln_b, eps) if ln_w is not None else pre
    return x * tokens.ne(padding_idx)[..., None].double(), pre


def embed_msa_64(tokens, table, pos_table, msa_pos, ln_w, ln_b, padding_idx: int, eps: float = 1e-5):
    """esm/model/msa_transformer.py:155-172 in float64: tokens [B,R,C]; msa_pos None or [>= R, E or 1] (row r of the
    alignment takes msa_pos[r]).  Returns (x [B,R,C,E], the rows before the LayerNorm)."""
    B, R, C = tokens.shape
    pre = table.double()[tokens] + pos_table.double()[positions(tokens, padding_idx)]
    if msa_pos is not None:
        pre = pre + msa_pos.double()[None, :R, None, :]
    x = layer_norm64(pre, ln_w, ln_b, eps)
    return x * tokens.ne(padding_idx)[..., None].double(), pre


def row_cond(pre: torch.Tensor, tokens: torch.Tensor, padding_idx: int) -> float:
    """max over the non-pad rows of |mean| / std: the conditioning ln_tol takes (a pad row may be constant; its output
    is multiplied by zero)"""
    c = pre.mean(-1).abs() / pre.std(-1, unbiased=False).clamp_min(1e-30)
    return float(c[tokens.ne(padding_idx)].max())


# ---- mean pool and log-softmax rows ---------------------------------------------------------------------------------
def mean_pool64(x: torch.Tensor, lengths: torch.Tensor) -> torch.Tensor:
    """scripts/extract.py:116-119 in float64: out[b] = x[b, 1 : 1 + n].mean(0) with n = lengths[b] clamped to
    [0, T - 1] (the slice's own clamp); NaN for the empty slice.  x [B,T,E] -> [B,E]."""
    B, T, E = x.shape
    rows = []
    for b in range(B):
        n = min(max(int(lengths[b]), 0), T - 1)
        rows.append(x[b, 1:1 + n].double().mean(0))
    return torch.stack(rows)


def mean_pool_bound(x: torch.Tensor, lengths: torch.Tensor) -> torch.Tensor:
    """|out - mean_pool64|: an n-term fp32 sum in any order (sum_bound), then 1 / n and the product (2 u |mean|)"""
    B, T, E = x.shape
    rows = []
    for b in range(B):
        n = min(max(int(lengths[b]), 0), T - 1)
        a = x[b, 1:1 + n].double().abs().sum(0)
        rows.append((sum_bound(a, max(n, 1)) + 2 * U32 * a) / max(n, 1))
    return torch.stack(rows) + 1e-45


def log_softmax64(x: torch.Tensor) -> torch.Tensor:
    """x - max - log sum exp(x - max) over the last dim in float64; -inf stays -inf, a row of -inf only is NaN"""
    x = x.double()
    m = x.amax(-1, keepdim=True)
    return (x - m) - torch.log(torch.exp(x - m).sum(-1, keepdim=True))


def log_softmax_bound(x: torch.Tensor) -> torch.Tensor:
    """|out - log_softmax64| for the fp32 kernel: x - m and the last subtraction are a rounding each of at most
    u (|x - m| + |lse|); expf (2 ulp), the sum (two terms per lane, five butterfly levels) and logf (1 ulp of |lse|)
    move lse by at most 9 u + u |lse|, taken as 16 u absolute (s >= 1: lse >= 0 is well conditioned)."""
    x = x.double()
    m = x.amax(-1, keepdim=True)
    lse = torch.log(torch.exp(x - m).sum(-1, keepdim=True))
    d = (x - m).abs()
    d = torch.where(torch.isinf(d), torch.zeros_like(d), d)
    return U32 * (2 * d + 2 * lse.abs() + 16)


# ---- standalone contact pass ----------------------------------------------------------------------------------------
def contact_stripes(attn: torch.Tensor, w: torch.Tensor, keep: Optional[torch.Tensor], lo: int, hi: int):
    """One layer's share of the accumulators of esmb200_contact_accumulate, float64: attn [B,H,T,T], w [H] ->
    (acc [B,S,S] = sum_h w_h A_h, row_sum [B,H,S], col_part [B,H,ceil(S/16),S]: the column sums of each stripe of 16
    cropped query rows).  row_sum[:, :, None] and col_part feed contacts_from_partials like the fused pass's partials."""
    a = masked_maps(attn, keep, lo, hi)[:, :, lo:hi, lo:hi]
    B, H, S, _ = a.shape
    acc = torch.einsum("bhij,h->bij", a, w.double().to(a.device))
    nt = (S + 15) // 16
    ap = torch.nn.functional.pad(a, [0, 0, 0, 16 * nt - S])
    return acc, a.sum(-1), ap.reshape(B, H, nt, 16, S).sum(3)


# ---- one transformer layer ------------------------------------------------------------------------------------------
def layer64(x: torch.Tensor, sd: Dict[str, torch.Tensor], pre: str, H: int, pad: torch.Tensor):
    """oracle.esm2_oracle.transformer_layer kept in float64 throughout (the oracle's softmax runs in fp32, as the
    reference's does), at any even head width d = E / H (the rotation pairs dimension j with j + d/2 under table column
    j < d/2, whatever d): x [B,T,E] float64, sd float64, pad [B,T] bool -> (x', probabilities [B,H,T,T])"""
    from oracle import esm2_oracle as o
    F = torch.nn.functional
    B, T, E = x.shape
    d = E // H
    assert d * H == E and d % 2 == 0
    h = o.layer_norm(x, sd[pre + "self_attn_layer_norm.weight"], sd[pre + "self_attn_layer_norm.bias"])
    a = pre + "self_attn."
    q = (F.linear(h, sd[a + "q_proj.weight"], sd[a + "q_proj.bias"]) * d ** -0.5).view(B, T, H, d).transpose(1, 2)
    k = F.linear(h, sd[a + "k_proj.weight"], sd[a + "k_proj.bias"]).view(B, T, H, d).transpose(1, 2)
    v = F.linear(h, sd[a + "v_proj.weight"], sd[a + "v_proj.bias"]).view(B, T, H, d).transpose(1, 2)
    cos, sin = o.rope_tables(sd[a + "rot_emb.inv_freq"], T)
    assert cos.shape == (T, d // 2)
    q, k = o.apply_rope(q, cos, sin), o.apply_rope(k, cos, sin)
    s = (q @ k.transpose(-1, -2)).masked_fill(pad[:, None, None, :], float("-inf"))
    p = torch.softmax(s, -1)
    ctx = (p @ v).transpose(1, 2).reshape(B, T, E)
    x = x + F.linear(ctx, sd[a + "out_proj.weight"], sd[a + "out_proj.bias"])
    h = o.layer_norm(x, sd[pre + "final_layer_norm.weight"], sd[pre + "final_layer_norm.bias"])
    h = o.gelu(F.linear(h, sd[pre + "fc1.weight"], sd[pre + "fc1.bias"]))
    return x + F.linear(h, sd[pre + "fc2.weight"], sd[pre + "fc2.bias"]), p
