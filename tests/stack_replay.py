"""Layer-by-layer replay of the library's layer stacks through the single-kernel C-ABI entry points, with every
intermediate kept, and the float64 checks of each stage on its own inputs (tests/test_gpu_stack_stages.py).

The replay packs the weights itself from the module parameters (`.half()`, esmb200_convert_split hi | lo, [Wq;Wk;Wv]
quantised by esmb200_quantize_fp8), heads of any width into zero-padded 64-wide slots by its own map
(kernel_refs.slot_columns), and takes every parameter from the reference's definition rather than from the library: the
module's LayerNorm eps, the q scale fp32(d ** -0.5) (fp32(d ** -0.5 / sqrt(R)) for the MSA row attention), and the
rotary tables of rotary_embedding.py:47-61, padded past d/2 with other values than the library's.  A stack that packs,
scales or wires one of them differently gives other bits than the replay.

  * pack_esm / replay_esm: one ESM-2 / ESM-1b layer in precision 0 (fp16), 1 (fp32x3) or 2 (fp8) at any head width,
    the QKV projection through esmb200_gemm_qkv_heads (the layer's own launch);
  * check_esm_stages / check_fp8_stages: each stage of one replayed layer against float64, worst ratios per stage;
  * pack_axial / replay_axial / check_axial_stages: one MSA Transformer AxialTransformerLayer in fp16 or fp32x3, and its
    stages against float64;
  * packed_arena: the bytes esmb200_layer_offload writes (api.cu packed_layout) at any head width.
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional

import numpy as np
import torch

import fp8_refs
import kernel_refs as kr


def P(t: Optional[torch.Tensor]):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def S():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def lib():
    from esm_b200 import _lib
    return _lib.load()


def check(rc):
    from esm_b200 import _lib
    _lib.check(rc)


def q_scale(d: int, rows: int = 0) -> float:
    """The reference's q scale as the fp32 value `q *= scaling` multiplies by: head_dim ** -0.5 (multihead_attention.py
    :100), or for the MSA row attention head_dim ** -0.5 / math.sqrt(num_rows) (axial_attention.py:36-38), both Python
    doubles rounded to fp32."""
    s = d ** -0.5
    if rows:
        s = s / math.sqrt(rows)
    return float(np.float32(s))


def rope_ref(inv_freq: torch.Tensor, T: int):
    """rotary_embedding.py:47-61 on the device: cos / sin of t * inv_freq, the first d/2 columns of the reference's
    duplicated table ([T, 32] for d = 64)"""
    t = torch.arange(T, device=inv_freq.device).type_as(inv_freq)
    freqs = torch.einsum("i,j->ij", t, inv_freq)
    emb = torch.cat((freqs, freqs), dim=-1)
    h = inv_freq.numel()
    return emb.cos()[:, :h].contiguous(), emb.sin()[:, :h].contiguous()


# the replay's table columns past d/2: other values than model.rope_tables' padding (cos 1, sin 0), so that a stack
# equal to the replay bit for bit rotates only zero rows of its packed weights by them
PAD_COS, PAD_SIN = 0.5, 0.25


def rope_slots(cos: torch.Tensor, sin: torch.Tensor, slots: int):
    """the reference's [T, d/2] tables widened to the QKV epilogue's [T, 32 * slots], columns past d/2 PAD_COS and
    PAD_SIN"""
    T, h = cos.shape
    c = torch.full((T, 32 * slots), PAD_COS, dtype=cos.dtype, device=cos.device)
    s = torch.full((T, 32 * slots), PAD_SIN, dtype=cos.dtype, device=cos.device)
    c[:, :h], s[:, :h] = cos, sin
    return c, s


def split_dev(w: torch.Tensor) -> torch.Tensor:
    """esmb200_convert_split: fp32 [N, K] -> fp16 [N, 2K] hi | lo"""
    w = w.detach().float().contiguous()
    N, K = w.shape
    out = torch.empty(N, 2 * K, dtype=torch.float16, device=w.device)
    check(lib().esmb200_convert_split(P(w), P(out), N, K, S()))
    return out


def _pack_matrix(w: torch.Tensor, precision: int):
    if precision == 1:
        return split_dev(w)
    return w.detach().half().contiguous()


# ---- ESM-2 / ESM-1b layer -------------------------------------------------------------------------------------------
def pack_esm(layer, precision: int) -> Dict:
    """The GEMM operands of one TransformerLayer at any head width d = E / H: [Wq;Wk;Wv] rows, their bias and out_proj's
    columns in zero-padded 64-wide head slots by the test's own map (kernel_refs.slot_columns; the identity at d = 64),
    fc1 and fc2 as they are.  The slot-packed fp32 matrices are then rounded to fp16, split by esmb200_convert_split
    (hi | lo, out_proj's pitch 2 Ea) or quantised by esmb200_quantize_fp8 in 128-row blocks over the zero rows too.
    Also returns the maps: rows [3E] (kernel_refs.slot_rows), cols [E], and Ea, slots."""
    a = layer.self_attn
    E, H = layer.embed_dim, layer.attention_heads
    slots = kr.head_slots(E, H)
    Ea = 64 * slots * H
    dev = a.q_proj.weight.device
    cols, rows = kr.slot_columns(E // H, H).to(dev), kr.slot_rows(E // H, H).to(dev)
    wqkv = torch.zeros(3 * Ea, E, device=dev)
    wqkv[rows] = torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight]).detach().float()
    bqkv = torch.zeros(3 * Ea, device=dev)
    bqkv[rows] = torch.cat([a.q_proj.bias, a.k_proj.bias, a.v_proj.bias]).detach().float()
    wo = torch.zeros(E, Ea, device=dev)
    wo[:, cols] = a.out_proj.weight.detach().float()
    pk = dict(b_qkv=bqkv, w_out=_pack_matrix(wo, 1 if precision == 1 else 0), rows=rows, cols=cols, Ea=Ea,
              slots=slots)
    if precision == 2:
        pk["q_qkv"], pk["s_qkv"] = fp8_refs.quantize_dev(wqkv, 128)
        pk["q_fc1"], pk["s_fc1"] = fp8_refs.quantize_dev(layer.fc1.weight.detach().float().contiguous(), 128)
        pk["q_fc2"], pk["s_fc2"] = fp8_refs.quantize_dev(layer.fc2.weight.detach().float().contiguous(), 128)
    else:
        pk["w_qkv"] = _pack_matrix(wqkv, precision)
        pk["w_fc1"] = _pack_matrix(layer.fc1.weight, precision)
        pk["w_fc2"] = _pack_matrix(layer.fc2.weight, precision)
    return pk


def _ln(x, ln, out, precision, scales=None):
    M, E = x.shape
    L = lib()
    if precision == 2:
        check(L.esmb200_layernorm_fp8(P(x), P(ln.weight), P(ln.bias), P(out), P(scales), M, E, ln.eps, S()))
    else:
        fn = L.esmb200_layernorm_split if precision == 1 else L.esmb200_layernorm_f16
        check(fn(P(x), P(ln.weight), P(ln.bias), P(out), M, E, ln.eps, S()))


def _gemm(epi, a, w, bias, out, M, N, K, precision, cos=None, sin=None, T=0, E=0):
    fn = lib().esmb200_gemm_split if precision == 1 else lib().esmb200_gemm_f16
    check(fn(epi, P(a), P(w), P(bias), P(out), M, N, K, P(cos), P(sin), T, E, S()))


def _gemm8(epi, a, sa, w, sw, bias, out, out_s, M, N, K, cos=None, sin=None, T=0, E=0):
    check(lib().esmb200_gemm_fp8(epi, P(a), P(sa), P(w), P(sw), P(bias), P(out), P(out_s), M, N, K, P(cos), P(sin), T, E,
                                 S()))


def replay_esm(layer, pk: Dict, x: torch.Tensor, pad8: torch.Tensor, B: int, T: int, cos, sin, precision: int,
               probs: Optional[torch.Tensor] = None) -> Dict:
    """One layer in place on x fp32 [B*T, E], kernel by kernel as api.cu attention_block / ffn_block launch them, at
    any head width.  cos, sin: the reference's [T, d/2] tables (rope_ref), widened by rope_slots for the QKV epilogue;
    None: no rotary embedding (ESM-1b).  probs: fp32 [B,H,T,T] to fill, or None.  Returns the stages: x0 (input), xn1,
    qkv, ctx (head-slot layout), x1 (after out_proj), xn2, h, x (output), the fp8 scales xs1 / xs2 / hs."""
    E, H, F = layer.embed_dim, layer.attention_heads, layer.ffn_embed_dim
    Ea, slots = pk["Ea"], pk["slots"]
    M = B * T
    pf = 2 if precision == 1 else 1
    dev = x.device
    L = lib()
    st = dict(x0=x.clone())
    if precision == 2:
        xn = torch.empty(M, E, dtype=torch.uint8, device=dev)
        xs = torch.empty((E + 127) // 128, M, device=dev)
    else:
        xn, xs = torch.empty(M, pf * E, dtype=torch.float16, device=dev), None
    _ln(x, layer.self_attn_layer_norm, xn, precision, xs)
    st.update(xn1=xn.clone(), xs1=None if xs is None else xs.clone())
    qkv = torch.empty(M, pf * 3 * Ea, dtype=torch.float16, device=dev)
    c, s_ = rope_slots(cos, sin, slots) if cos is not None else (None, None)
    w, ws = (pk["q_qkv"], pk["s_qkv"]) if precision == 2 else (pk["w_qkv"], None)
    check(L.esmb200_gemm_qkv_heads(precision, P(xn), P(xs), P(w), P(ws), P(pk["b_qkv"]), P(qkv), M, E, H,
                                   q_scale(E // H), P(c), P(s_), T if cos is not None else 0, S()))
    st["qkv"] = qkv.clone()
    ctx = torch.empty(M, pf * Ea, dtype=torch.float16, device=dev)
    scratch = torch.empty(L.esmb200_attention_scratch_bytes(B, T), dtype=torch.uint8, device=dev)
    att = (L.esmb200_attention_split if precision == 1 else
           L.esmb200_attention128 if slots == 2 else L.esmb200_attention)
    check(att(P(qkv), P(pad8), P(ctx), P(probs), B, T, H, P(scratch), S()))
    st["ctx"] = ctx.clone()
    _gemm(kr.EPI_BIAS_RESIDUAL, ctx, pk["w_out"], layer.self_attn.out_proj.bias, x, M, E, Ea,
          1 if precision == 1 else 0)
    st["x1"] = x.clone()
    _ln(x, layer.final_layer_norm, xn, precision, xs)
    st.update(xn2=xn.clone(), xs2=None if xs is None else xs.clone())
    if precision == 2:
        h = torch.empty(M, F, dtype=torch.uint8, device=dev)
        hs = torch.empty(F // 128, M, device=dev)
        _gemm8(fp8_refs_epi_gelu(), xn, xs, pk["q_fc1"], pk["s_fc1"], layer.fc1.bias, h, hs, M, F, E)
        st.update(h=h.clone(), hs=hs.clone())
        _gemm8(kr.EPI_BIAS_RESIDUAL, h, hs, pk["q_fc2"], pk["s_fc2"], layer.fc2.bias, x, None, M, E, F)
    else:
        h = torch.empty(M, pf * F, dtype=torch.float16, device=dev)
        _gemm(kr.EPI_BIAS_GELU, xn, pk["w_fc1"], layer.fc1.bias, h, M, F, E, precision)
        st["h"] = h.clone()
        _gemm(kr.EPI_BIAS_RESIDUAL, h, pk["w_fc2"], layer.fc2.bias, x, M, E, F, precision)
    st["x"] = x
    return st


def fp8_refs_epi_gelu() -> int:
    from esm_b200 import _lib
    return _lib.EPI_GELU_FP8


# ---- float64 stages -------------------------------------------------------------------------------------------------
def _worst(worst: Dict, name: str, ratio: float):
    assert ratio == ratio, f"NaN ratio in stage {name}"
    worst[name] = max(worst.get(name, 0.0), ratio)


def _ratio(err: torch.Tensor, bound: torch.Tensor) -> float:
    assert not bool(err.isnan().any()), "NaN in a stage"
    r = float((err / bound).max())
    assert r == r, "NaN ratio in a stage (a zero bound at a zero error)"
    return r


def _ln_stage(x, ln, got, split):
    """(error, bound) of a LayerNorm -> fp16 (or hi | lo) output against float64 on the kernel's fp32 input"""
    want, b = _ln_want(x, ln)
    E = x.shape[-1]
    if split:
        g = kr.join64(got[:, :E], got[:, E:])
        b = b + kr.split_rep_bound(want.abs() + b)
    else:
        g = got.double()
        b = b + kr.f16_bound(want.abs() + b)
    return (g - want).abs(), b


def _ln_want(x, ln):
    """(float64 LayerNorm of the kernel's fp32 input, the fp32 kernel's bound ln_tol at the row's |mean|/std)"""
    E = x.shape[-1]
    xd = x.double()
    want = kr.layer_norm64(xd, ln.weight, ln.bias, ln.eps)
    cond = (xd.mean(-1, keepdim=True).abs() / xd.std(-1, unbiased=False, keepdim=True).clamp_min(1e-30))
    return want, kr.ln_tol(E, cond) * kr.ln_scale(want, ln.weight, ln.bias)


def ln_stage(worst, name, x, ln, got, split):
    err, b = _ln_stage(x, ln, got, split)
    _worst(worst, name, _ratio(err, b))


def _heads(t: torch.Tensor, B: int, T: int, H: int, i: int, slots: int = 1) -> torch.Tensor:
    """section i (0 q, 1 k, 2 v) of the head-slot layout [B*T, 3 Ea] (Ea = 64 slots H) as [B, H, T, 64 slots]"""
    D = 64 * slots
    Ea = D * H
    return t[:, i * Ea:(i + 1) * Ea].reshape(B, T, H, D).transpose(1, 2)


def padding_columns(rows: torch.Tensor, width: int) -> torch.Tensor:
    """[width] bool: the columns of a head-slot tensor that no reference column maps to"""
    m = torch.ones(width, dtype=torch.bool, device=rows.device)
    m[rows] = False
    return m


def zero_columns_stage(name, t, rows, n_halves=1):
    """every padding column of the head-slot tensor t ([M, W] or [M, n_halves W] hi | lo) is exactly 0"""
    W = t.shape[1] // n_halves
    pad = padding_columns(rows, W)
    for i in range(n_halves):
        assert bool((t[:, i * W:(i + 1) * W][:, pad] == 0).all()), f"{name}: a padding column is not 0"


def qkv_stage(worst, xn, w_qkv, bqkv, qkv, E, H, qs, T, cos, sin, split, zero_rows=None):
    """the QKV projection (q scale, rotate-half RoPE when cos [T, d/2] is given) on the kernel's own operands, compared
    in the reference's layout: w_qkv [3Ea, K] and bqkv [3Ea] in head slots, the kernel's qkv [M, 3Ea] (hi | lo
    [M, 6Ea]) read through kernel_refs.slot_rows, against qkv_ref_heads on the unpadded rows; every padding column
    exactly 0.  zero_rows [M] bool: rows whose q the caller zeroed (the MSA row attention's padded tokens)."""
    rows = kr.slot_rows(E // H, H).to(qkv.device)
    if split:
        zero_columns_stage("qkv", qkv, rows, 2)
        Ea3 = qkv.shape[1] // 2
        xh, xl, wh, wl = xn[:, :E], xn[:, E:], w_qkv[rows, :E], w_qkv[rows, E:]
        aj, wj = kr.join64(xh, xl), kr.join64(wh, wl)
        b = bqkv[rows]
        y_pre = aj @ wj.t() + b.double()
        y_pre[:, :E] *= qs
        y, _ = kr.qkv_ref_heads(aj, wj, b, qs, H, T, cos, sin)
        bnd = split_qkv_heads_bound(xh, xl, wh, wl, y_pre, E, H, qs, cos is not None) + kr.split_rep_bound(y)
        got = kr.join64(qkv[:, :Ea3][:, rows], qkv[:, Ea3:][:, rows])
    else:
        zero_columns_stage("qkv", qkv, rows)
        y, absdot = kr.qkv_ref_heads(xn, w_qkv[rows], bqkv[rows], qs, H, T, cos, sin)
        bnd = kr.qkv_bound(y, absdot, E)
        got = qkv[:, rows].double()
    if zero_rows is not None:
        y[zero_rows, :E] = 0.0
    _worst(worst, "qkv", _ratio((got - y).abs(), bnd))


def split_qkv_heads_bound(ah, al, wh, wl, y_pre, E, H, q_scale, rotary):
    """test_gpu_gemm_split.split_qkv_bound in the reference's layout at head width d = E / H: the split GEMM's
    accumulation bound, times q_scale on the q columns plus one rounding (u |y_pre|), and for the rotate-half pairs
    (j, j + d/2) of the q and k heads both members' bounds plus the rotation's two products and one add
    (4 u (|x1| + |x2|)).  y_pre: the unrotated (a w^T + bias) * scale in float64."""
    b = kr.split_acc_bound(ah, al, wh, wl, E, y_pre)
    b[:, :E] *= q_scale
    b = b + kr.U32 * y_pre.abs()
    if rotary:
        x = kr.rope_pair_sum(y_pre.abs(), E, H)
        b = kr.rope_pair_sum(b, E, H)
        b[:, :2 * E] += 4 * kr.U32 * x[:, :2 * E]
    return b


def key_blocks(slots: int):
    """the key-block size of the fp16 forward kernel: 128 (attention_wg_kernel) for one slot per head, 64
    (attention_fwd_kernel<false, 2>, esmb200_attention128) for two"""
    return (128,) if slots == 1 else (64,)


def attention_stage_f16(worst, qkv, ctx, pad, B, T, H, probs=None, blocks=(128,), prefix="", slots=1, qrows=None):
    """fp16 attention on the kernel's q, k, v (qkv [B*T, 3Ea] in head slots, sequences of T tokens, pad [B, T] bool):
    ctx element-wise (attn_ctx_bound) and per (sequence, head) rel-Fro (attn_relfro_gate), probabilities [B, H, T, T]
    and row sums at the query rows qrows [B, T] bool (None: the valid ones, ~pad).  The heads are taken 64 slots wide,
    their padding columns included (zeros add nothing to q k^T or P v).  blocks: the key-block sizes the kernel may
    walk; every bound is the largest over them."""
    q, k, v = (_heads(qkv, B, T, H, i, slots) for i in range(3))
    got = _heads(ctx, B, T, H, 0, slots).double()
    if qrows is None:
        qrows = ~pad.bool()
    terms = {bl: [0, 0, 0] for bl in blocks}
    err2 = 0
    for i0, r0 in kr.attention64_rows(q, k, v, pad, blocks[0]):
        rs = [r0] + [kr.attention64(q[..., i0:i0 + r0["ctx"].shape[-2], :], k, v, pad, bl) for bl in blocks[1:]]
        n = r0["ctx"].shape[-2]
        g = got[..., i0:i0 + n, :]
        e = (g - r0["ctx"]).abs()
        _worst(worst, prefix + "ctx", _ratio(e, torch.stack([kr.attn_ctx_bound(r) for r in rs]).amax(0)))
        for bl, r in zip(blocks, rs):
            t = kr.attn_relfro_terms(r)
            terms[bl] = [a + b for a, b in zip(terms[bl], t)]
        err2 = err2 + e.pow(2).sum((-1, -2))
        if probs is not None:
            rows = qrows[:, i0:i0 + n]
            m = rows[:, None, :, None].expand_as(r0["p"])
            pr = probs[:, :, i0:i0 + n].double()
            pb = torch.stack([kr.attn_probs_bound(r) for r in rs]).amax(0)
            _worst(worst, prefix + "probs", _ratio((pr - r0["p"]).abs()[m], pb[m]))
            mr = rows[:, None, :].expand(B, H, n)
            rb = torch.stack([kr.attn_rowsum_bound(r) for r in rs]).amax(0)
            _worst(worst, prefix + "rowsum", _ratio((pr.sum(-1) - 1).abs()[mr], rb[mr]))
        del rs, r0
    gate = torch.stack([kr.attn_relfro_combine(*terms[bl]) for bl in blocks]).amax(0)
    ctx2 = terms[blocks[0]][2]
    live = ctx2 > 0  # a sequence of padding only has ctx 0, written as 0 (checked element-wise above)
    fro = err2.sqrt() / ctx2.sqrt().clamp_min(1e-300)
    _worst(worst, prefix + "ctx_relfro_gate", float((fro[live] / gate[live]).max()))


def attention_stage_split(worst, qkv, ctx, pad, B, T, H, probs=None, prefix="", qrows=None):
    """fp32x3 attention on the kernel's q, k, v hi | lo (qkv [B*T, 6E]): the split attention tests' element bound and
    per-head gate, and the probabilities (test_gpu_attention_split.probs_bound) and row sums (kernel_refs
    .attn_rowsum_bound on the split reference) at the query rows qrows [B, T] bool (None: ~pad)"""
    import test_gpu_attention_split as tas
    E = 64 * H
    r = tas.reference(qkv[:, :3 * E], qkv[:, 3 * E:], pad, B, T, H)
    got = _heads(ctx[:, :E].double(), B, T, H, 0) + _heads(ctx[:, E:].double(), B, T, H, 0)
    err = (got - r["ctx"]).abs()
    _worst(worst, prefix + "ctx", _ratio(err, tas.ctx_bound(r)))
    fro = (err.pow(2).sum((-1, -2)) / r["ctx"].pow(2).sum((-1, -2)).clamp_min(1e-300)).sqrt()
    _worst(worst, prefix + "ctx_relfro_gate", float((fro / tas.relfro_gate(r)).max()))
    if probs is not None:
        if qrows is None:
            qrows = ~pad.bool()
        m = qrows[:, None, :, None].expand_as(r["p"])
        pr = probs.double()
        _worst(worst, prefix + "probs", _ratio((pr - r["p"]).abs()[m], tas.probs_bound(r)[m]))
        mr = qrows[:, None, :].expand(B, H, T)
        _worst(worst, prefix + "rowsum", _ratio((pr.sum(-1) - 1).abs()[mr], kr.attn_rowsum_bound(r)[mr]))


def column_query_rows(cpad: torch.Tensor) -> torch.Tensor:
    """[N, R] bool from the column sequences' key padding cpad [N, R]: every query row of a column with at least one
    valid key.  The column attention masks keys only and keeps q at padded rows (axial_attention.py:211-217, no
    zeroed rows in the stack), so a padded query row of a live column is a softmax row over the valid keys like any
    other.  A column of padding only is written as 0 (the reference gives 1/R there) and is checked for that alone
    (column_zero_stage)."""
    return (~cpad.bool()).any(-1, keepdim=True).expand_as(cpad)


def column_zero_stage(name: str, probs: torch.Tensor, cpad: torch.Tensor):
    """the exact zeros of the column maps probs [N, H, R, R] under the key padding cpad [N, R]: every padded key of
    every row, and every entry of a column whose keys are all padding"""
    km = cpad.bool()[:, None, None, :].expand_as(probs)
    assert bool((probs[km] == 0).all()), f"{name}: a padded key has probability"
    dead = ~column_query_rows(cpad)[:, 0]
    assert bool((probs[dead] == 0).all()), f"{name}: a column of padding only is not 0"


def residual_stage(worst, name, a_op, w_op, bias, x_in, x_out, K, split):
    """x_out = x_in + a w^T + bias (fp16 or hi | lo operands) within residual_bound"""
    if split:
        ah, al, wh, wl = a_op[:, :K], a_op[:, K:], w_op[:, :K], w_op[:, K:]
        upd = kr.join64(ah, al) @ kr.join64(wh, wl).t() + bias.double()
        acc = kr.split_acc_bound(ah, al, wh, wl, K, upd)
    else:
        upd, absdot = kr.gemm_exact(a_op, w_op, bias)
        acc = kr.gemm_acc_bound(absdot, K, upd)
    want = x_in.double() + upd
    _worst(worst, name, _ratio((x_out.double() - want).abs(), kr.residual_bound(acc, want)))


def fc1_stage(worst, xn, w, bias, h, E, F, split):
    """h = GELU(xn w^T + bias) in fp16 or hi | lo: 1.13 x the GEMM bound (|GELU'| <= 1.13), gelu_bound, output rounding"""
    if split:
        ah, al, wh, wl = xn[:, :E], xn[:, E:], w[:, :E], w[:, E:]
        y = kr.join64(ah, al) @ kr.join64(wh, wl).t() + bias.double()
        acc = kr.split_acc_bound(ah, al, wh, wl, E, y)
        got = kr.join64(h[:, :F], h[:, F:])
        want = kr.gelu64(y)
        b = 1.13 * acc + kr.gelu_bound(y) + kr.split_rep_bound(want.abs() + 1.13 * acc)
    else:
        y, absdot = kr.gemm_exact(xn, w, bias)
        acc = kr.gemm_acc_bound(absdot, E, y)
        got = h.double()
        want = kr.gelu64(y)
        b = 1.13 * acc + kr.gelu_bound(y) + kr.f16_bound(want.abs() + 1.13 * acc)
    _worst(worst, "fc1", _ratio((got - want).abs(), b))


def check_esm_stages(layer, pk: Dict, st: Dict, pad: torch.Tensor, B: int, T: int, cos, precision: int, worst: Dict,
                     probs: Optional[torch.Tensor] = None, sin=None):
    """Every stage of one replayed layer against float64 on that stage's own inputs; the largest error / bound of each
    stage is folded into `worst`.  fp16 and fp32x3 (fp8: check_fp8_stages).  cos, sin: the reference's [T, d/2]
    tables.  The QKV stage runs in the reference's layout, attention and out_proj (K = Ea) on the head slots."""
    E, H, F = layer.embed_dim, layer.attention_heads, layer.ffn_embed_dim
    split = precision == 1
    a = layer.self_attn
    ln_stage(worst, "ln1", st["x0"], layer.self_attn_layer_norm, st["xn1"], split)
    ln_stage(worst, "ln2", st["x1"], layer.final_layer_norm, st["xn2"], split)
    qkv_stage(worst, st["xn1"], pk["w_qkv"], pk["b_qkv"], st["qkv"], E, H, q_scale(E // H), T, cos, sin, split)
    zero_columns_stage("ctx", st["ctx"], pk["cols"], 2 if split else 1)
    if split:
        attention_stage_split(worst, st["qkv"], st["ctx"], pad, B, T, H, probs)
    else:
        attention_stage_f16(worst, st["qkv"], st["ctx"], pad, B, T, H, probs, key_blocks(pk["slots"]), slots=pk["slots"])
    residual_stage(worst, "out_proj", st["ctx"], pk["w_out"], a.out_proj.bias, st["x0"], st["x1"], pk["Ea"], split)
    fc1_stage(worst, st["xn2"], pk["w_fc1"], layer.fc1.bias, st["h"], E, F, split)
    residual_stage(worst, "fc2", st["h"], pk["w_fc2"], layer.fc2.bias, st["x1"], st["x"], F, split)


# ---- fp8 stages (fp8_refs' bounds on the dequantised operands) -----------------------------------------------------
def _e4m3(q: torch.Tensor) -> torch.Tensor:
    return q.view(torch.float8_e4m3fn)


def _codes_stage(worst, name, q8, s, y, ybnd):
    """an e4m3 output with its 1 x 128 scales against float64 (fp8_refs.check_codes): no scale off by more than the
    edge case, no code farther from y than half an e4m3 ulp plus the bound, boundary flips under 2 %"""
    r = fp8_refs.check_codes(_e4m3(q8), s, y, ybnd, device=y.device)
    assert r["bad_scale"] == 0 and r["bad_code"] == 0 and r["flips"] <= max(64, r["n"] // 50), (name, r)
    _worst(worst, name + "_flip_share", r["flips"] / r["n"])


def check_fp8_stages(layer, pk: Dict, st: Dict, pad: torch.Tensor, B: int, T: int, cos, sin, worst: Dict,
                     probs: Optional[torch.Tensor] = None):
    """The stages of one replayed fp8 layer: LayerNorm -> e4m3 codes and scales, the QKV, fc1 (GELU -> e4m3) and fc2
    (residual) GEMMs on the dequantised operands with fp8_refs.acc_bound (2^-11 per K block), and the stages the fp8
    layer shares with fp16 (attention, out_proj)."""
    E, H, F = layer.embed_dim, layer.attention_heads, layer.ffn_embed_dim
    a = layer.self_attn
    for name, x, ln, q8, s in (("ln1_codes", st["x0"], layer.self_attn_layer_norm, st["xn1"], st["xs1"]),
                               ("ln2_codes", st["x1"], layer.final_layer_norm, st["xn2"], st["xs2"])):
        want, b = _ln_want(x, ln)
        _codes_stage(worst, name, q8, s, want, b + 2.0 ** -24 * want.abs())
    # the QKV projection in the reference's layout (the dequantised slot rows of the reference's rows, K = E); the
    # quantisation's zero rows must give exactly 0
    rows = pk["rows"]
    zero_columns_stage("qkv", st["qkv"], rows)
    A = fp8_refs.dequantize(_e4m3(st["xn1"]), st["xs1"], 1)
    W = fp8_refs.dequantize(_e4m3(pk["q_qkv"]), pk["s_qkv"], 128)[rows]
    y, absdot = kr.qkv_ref_heads(A, W, pk["b_qkv"][rows], q_scale(E // H), H, T, cos, sin)
    acc = absdot * (2.0 ** -11 + 2.0 ** -24 * math.ceil(E / 128))
    got = st["qkv"][:, rows].double()
    _worst(worst, "qkv", _ratio((got - y).abs(), acc + 6 * kr.U32 * y.abs() + kr.f16_bound(y)))
    del A, W, y, absdot, acc, got
    zero_columns_stage("ctx", st["ctx"], pk["cols"])
    attention_stage_f16(worst, st["qkv"], st["ctx"], pad, B, T, H, probs, key_blocks(pk["slots"]), slots=pk["slots"])
    residual_stage(worst, "out_proj", st["ctx"], pk["w_out"], a.out_proj.bias, st["x0"], st["x1"], pk["Ea"], False)
    A = fp8_refs.dequantize(_e4m3(st["xn2"]), st["xs2"], 1)
    W = fp8_refs.dequantize(_e4m3(pk["q_fc1"]), pk["s_fc1"], 128)
    ref = A @ W.t() + layer.fc1.bias.double()
    y = kr.gelu64(ref)
    ybnd = 1.13 * fp8_refs.acc_bound(A, W) + 1e-7 * ref.abs() + 2.0 ** -20 * y.abs()
    _codes_stage(worst, "fc1_codes", st["h"], st["hs"], y, ybnd)
    del A, W, ref, y, ybnd
    A = fp8_refs.dequantize(_e4m3(st["h"]), st["hs"], 1)
    W = fp8_refs.dequantize(_e4m3(pk["q_fc2"]), pk["s_fc2"], 128)
    upd = A @ W.t() + layer.fc2.bias.double()
    want = st["x1"].double() + upd
    acc = fp8_refs.acc_bound(A, W) + 2 * kr.U32 * upd.abs()
    _worst(worst, "fc2", _ratio((st["x"].double() - want).abs(), kr.residual_bound(acc, want)))


# ---- MSA Transformer axial layer ------------------------------------------------------------------------------------
def pack_axial(layer, precision: int) -> Dict:
    out = {}
    for key, blk in (("row", layer.row_self_attention.layer), ("col", layer.column_self_attention.layer)):
        w = torch.cat([blk.q_proj.weight, blk.k_proj.weight, blk.v_proj.weight]).detach().float().contiguous()
        out[key + "_qkv"] = _pack_matrix(w, precision)
        out[key + "_b"] = torch.cat([blk.q_proj.bias, blk.k_proj.bias, blk.v_proj.bias]).detach().float().contiguous()
        out[key + "_out"] = _pack_matrix(blk.out_proj.weight, precision)
    ffn = layer.feed_forward_layer.layer
    out["fc1"], out["fc2"] = _pack_matrix(ffn.fc1.weight, precision), _pack_matrix(ffn.fc2.weight, precision)
    return out


def replay_axial(layer, pk: Dict, x: torch.Tensor, pad: Optional[torch.Tensor], B: int, R: int, C: int,
                 precision: int, row_probs: Optional[torch.Tensor] = None) -> Dict:
    """One AxialTransformerLayer in place on x fp32 [B*R*C, E]: tied row attention (q zeroed at padded tokens, key
    padding from row 0 of each alignment), column attention, feed-forward.  pad [B,R,C] bool or None.  Returns the
    stages: x0, row_xn, row_qkv (q zeroed), row_ctx, x_row, col_xn, col_qkv, col_ctx, x_col, ffn_xn, h, x."""
    E, H, F = layer.embedding_dim, layer.num_heads, layer.ffn_embedding_dim
    M = B * R * C
    pf = 2 if precision == 1 else 1
    split = precision == 1
    dev = x.device
    L = lib()
    xn = torch.empty(M, pf * E, dtype=torch.float16, device=dev)
    qkv = torch.empty(M, pf * 3 * E, dtype=torch.float16, device=dev)
    ctx = torch.empty(M, pf * E, dtype=torch.float16, device=dev)
    key_pad = col_pad = None
    if pad is not None:
        key_pad = pad[:, 0].contiguous().to(torch.uint8)
        col_pad = pad.permute(0, 2, 1).contiguous().to(torch.uint8)
    st = dict(x0=x.clone())

    def qkv_proj(w, b, scale):
        if split:
            check(L.esmb200_gemm_qkv_split(P(xn), P(w), P(b), P(qkv), M, E, scale, S()))
        else:
            check(L.esmb200_gemm_qkv_f16(P(xn), P(w), P(b), P(qkv), M, E, scale, None, None, 0, S()))

    blk = layer.row_self_attention
    _ln(x, blk.layer_norm, xn, precision)
    st["row_xn"] = xn.clone()
    qkv_proj(pk["row_qkv"], pk["row_b"], q_scale(64, R))
    if pad is not None:
        q5 = qkv.view(B, R, C, 3 * pf, E)
        q5[:, :, :, 0].masked_fill_(pad[..., None], 0)
        if split:
            q5[:, :, :, 3].masked_fill_(pad[..., None], 0)
    st["row_qkv"] = qkv.clone()
    if split:
        nbytes, tied = L.esmb200_tied_row_attention_split_scratch_bytes(B, C, H), L.esmb200_tied_row_attention_split
    else:
        nbytes, tied = L.esmb200_tied_row_attention_scratch_bytes(B, C, H), L.esmb200_tied_row_attention
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    check(tied(P(qkv), P(key_pad), P(ctx), P(row_probs), B, R, C, H, P(scratch), nbytes, S()))
    st["row_ctx"] = ctx.clone()
    _gemm(kr.EPI_BIAS_RESIDUAL, ctx, pk["row_out"], blk.layer.out_proj.bias, x, M, E, E, precision)
    st["x_row"] = x.clone()
    blk = layer.column_self_attention
    _ln(x, blk.layer_norm, xn, precision)
    st["col_xn"] = xn.clone()
    qkv_proj(pk["col_qkv"], pk["col_b"], q_scale(64))
    st["col_qkv"] = qkv.clone()
    scratch = torch.empty(L.esmb200_attention_scratch_bytes(B * C, R), dtype=torch.uint8, device=dev)
    col = L.esmb200_column_attention_split if split else L.esmb200_column_attention
    check(col(P(qkv), P(col_pad), P(ctx), B, R, C, H, P(scratch), S()))
    st["col_ctx"] = ctx.clone()
    _gemm(kr.EPI_BIAS_RESIDUAL, ctx, pk["col_out"], blk.layer.out_proj.bias, x, M, E, E, precision)
    st["x_col"] = x.clone()
    blk = layer.feed_forward_layer
    _ln(x, blk.layer_norm, xn, precision)
    st["ffn_xn"] = xn.clone()
    h = torch.empty(M, pf * F, dtype=torch.float16, device=dev)
    _gemm(kr.EPI_BIAS_GELU, xn, pk["fc1"], blk.layer.fc1.bias, h, M, F, E, precision)
    st["h"] = h.clone()
    _gemm(kr.EPI_BIAS_RESIDUAL, h, pk["fc2"], blk.layer.fc2.bias, x, M, E, F, precision)
    st["x"] = x
    return st


def _column_major(t: torch.Tensor, B: int, R: int, C: int) -> torch.Tensor:
    """[B*R*C, w] row-major alignment tensor -> [B*C*R, w]: the column sequences of R tokens, one after another"""
    w = t.shape[-1]
    return t.view(B, R, C, w).permute(0, 2, 1, 3).reshape(B * C * R, w)


def check_axial_stages(layer, pk: Dict, st: Dict, pad: Optional[torch.Tensor], B: int, R: int, C: int,
                       precision: int, worst: Dict, col_probs: Optional[torch.Tensor] = None):
    """Every stage of one replayed AxialTransformerLayer against float64 on its own inputs: the three LayerNorms, the
    row and column QKV (row q scale fp32(d^-1/2 / sqrt(R)), q zero at padded tokens), the tied row attention end to
    end (tied_ctx_bound, tied_relfro_gate), the column attention (the fp16 or split attention bounds, per column
    sequence of R tokens, over both key-block sizes of the fp16 kernels), the two out-projections and the
    feed-forward.  col_probs: the layer's column maps fp32 [B, C, H, R, R] (the stack's), checked at every query row of
    every live column (column_query_rows) and exactly 0 where column_zero_stage says."""
    E, H, F = layer.embedding_dim, layer.num_heads, layer.ffn_embedding_dim
    split = precision == 1
    pf = 2 if split else 1
    ln_stage(worst, "row_ln", st["x0"], layer.row_self_attention.layer_norm, st["row_xn"], split)
    ln_stage(worst, "col_ln", st["x_row"], layer.column_self_attention.layer_norm, st["col_xn"], split)
    ln_stage(worst, "ffn_ln", st["x_col"], layer.feed_forward_layer.layer_norm, st["ffn_xn"], split)
    zero = pad.reshape(-1) if pad is not None else None
    w_sub = {}
    qkv_stage(w_sub, st["row_xn"], pk["row_qkv"], pk["row_b"], st["row_qkv"], E, H, q_scale(64, R), 1, None, None,
              split, zero)
    _worst(worst, "row_qkv", w_sub.pop("qkv"))
    qkv_stage(w_sub, st["col_xn"], pk["col_qkv"], pk["col_b"], st["col_qkv"], E, H, q_scale(64), 1, None, None, split)
    _worst(worst, "col_qkv", w_sub.pop("qkv"))
    # tied row attention on its own (q-zeroed) q, k, v
    key_pad = pad[:, 0] if pad is not None else None
    r = kr.tied64(st["row_qkv"], key_pad, B, R, C, H, split)
    cv = st["row_ctx"].double().view(B, R, C, pf * E)
    got = (cv[..., :E] + cv[..., E:] if split else cv).reshape(B, R, C, H, 64)
    err = (got - r["ctx"]).abs()
    _worst(worst, "tied_ctx", _ratio(err, kr.tied_ctx_bound(r)))
    fro = (err.pow(2).sum((1, 2, 4)) / r["ctx"].pow(2).sum((1, 2, 4)).clamp_min(1e-300)).sqrt()
    _worst(worst, "tied_relfro_gate", float((fro / kr.tied_relfro_gate(r)).max()))
    del r, err, got
    # column attention: B*C sequences of R tokens
    cq, cc = _column_major(st["col_qkv"], B, R, C), _column_major(st["col_ctx"], B, R, C)
    cpad = pad.permute(0, 2, 1).reshape(B * C, R) if pad is not None else torch.zeros(B * C, R, dtype=torch.bool,
                                                                                         device=cq.device)
    cp = qrows = None
    if col_probs is not None:
        cp = col_probs.view(B * C, H, R, R)
        column_zero_stage("col_probs", cp, cpad)
        qrows = column_query_rows(cpad)
    if split:
        attention_stage_split(worst, cq, cc, cpad, B * C, R, H, cp, prefix="col_", qrows=qrows)
    else:
        attention_stage_f16(worst, cq, cc, cpad, B * C, R, H, cp, blocks=(64, 128), prefix="col_", qrows=qrows)
    residual_stage(worst, "row_out_proj", st["row_ctx"], pk["row_out"], layer.row_self_attention.layer.out_proj.bias,
                   st["x0"], st["x_row"], E, split)
    residual_stage(worst, "col_out_proj", st["col_ctx"], pk["col_out"],
                   layer.column_self_attention.layer.out_proj.bias, st["x_row"], st["x_col"], E, split)
    ffn = layer.feed_forward_layer.layer
    fc1_stage(worst, st["ffn_xn"], pk["fc1"], ffn.fc1.bias, st["h"], E, F, split)
    residual_stage(worst, "fc2", st["h"], pk["fc2"], ffn.fc2.bias, st["x_col"], st["x"], F, split)


# ---- the packed matrices of esmb200_layer_offload -------------------------------------------------------------------
def _align(n: int, a: int = 1024) -> int:
    return (n + a - 1) // a * a


def packed_arena(layer, split: bool) -> torch.Tensor:
    """uint8 bytes of api.cu packed_layout for one TransformerLayer of any head width, built on the host from the
    module's parameters: [Wq;Wk;Wv] rows and out_proj columns in their zero-padded 64-wide head slots
    (fp8_refs.head_slot), fc1 and fc2 as they are; fp16, or with split the hi | lo halves side by side along K, each
    matrix 1024-byte aligned."""
    a = layer.self_attn
    E, H = layer.embed_dim, layer.attention_heads
    d = E // H
    Ea = 64 * kr.head_slots(E, H) * H
    slot = fp8_refs.head_slot(torch.arange(E), d)

    def enc(w32):  # fp32 [N, K] -> fp16 [N, K] or [N, 2K]
        w32 = w32.detach().float().cpu()
        if not split:
            return w32.half()
        hi, lo = kr.split16(w32)
        return torch.cat([hi, lo], 1)

    pf = 2 if split else 1
    qkv = torch.zeros(3 * Ea, pf * E, dtype=torch.float16)
    for s3, w in enumerate((a.q_proj.weight, a.k_proj.weight, a.v_proj.weight)):
        qkv[s3 * Ea + slot] = enc(w)
    out = torch.zeros(E, pf * Ea, dtype=torch.float16)
    wo = enc(a.out_proj.weight)
    out[:, slot] = wo[:, :E]
    if split:
        out[:, Ea + slot] = wo[:, E:]
    parts = [qkv, out, enc(layer.fc1.weight), enc(layer.fc2.weight)]
    chunks = []
    for p in parts:
        b = p.contiguous().view(torch.uint8).reshape(-1)
        chunks.append(torch.cat([b, torch.zeros(_align(b.numel()) - b.numel(), dtype=torch.uint8)]))
    return torch.cat(chunks)
