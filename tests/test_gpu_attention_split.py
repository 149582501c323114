"""GPU (-m gpu): the fp32x3 attention kernels against float64 softmax attention on q, k, v = hi + lo:
attention_fwd_kernel<true, 1> (csrc/attention8.cuh) through esmb200_attention_split and esmb200_column_attention_split,
and attention_probs_kernel<1> (csrc/attention_probs.cuh).  qkv is [M, 6E] = [q k v]_hi | [q k v]_lo, ctx [M, 2E] hi | lo.
The forward kernel walks 64-key blocks, so the block edges sit at T = 64, 128, ...; the probability kernel uses 128-key
tiles.  Sharp logits (std 8) are included wherever a dropped P_lo . V or q_lo . k term must show: P_lo carries weight
against the bound only when attention is concentrated.

Element bound on ctx (ctx_bound below), first order in the kernel's errors.  Each unnormalised weight e^(s_j - m) is off
by a relative Delta_j:
  * the logit: 3 passes x 4 k16 steps of truncating fp32 accumulation, (12 + 4) 2^-22 sum|q k| over the three passes,
    plus the dropped q_lo k_lo term;
  * ex2.approx (2 ulp: 2^-22, doubled) and the fp32 roundings of s log2(e) - m log2(e) (2^-23 (|s| + 3 |m|));
so ctx moves by sum_j p_j Delta_j (v_j - ctx) <= (p Delta) |v| + (sum_j p_j Delta_j) |ctx|.  Then the P . V accumulation
(12 nblk + 4) 2^-22 sum p|v| (three passes, nblk 64-key blocks into one accumulator), the hi | lo representation of P
(2^-21 p + 2^-25 / l per key, l = sum_j e^(s_j - m)), the per-block rescale of O (nblk u sum p|v|), the fp32 row sum,
its rescales and 1/l (18 nblk + 4) u |ctx|, and the output's own hi | lo representation (kr.split_rep_bound)."""
import ctypes

import pytest
import torch

import kernel_refs as kr
from test_gpu_attention_wg import _stats

pytestmark = pytest.mark.gpu

U = kr.U32
# Per-(sequence, head) rel-Frobenius gate in units of (12 nblk + 4) 2^-25 + 2^-23 max|s| (the P . V accumulation drift,
# and the relative weight error that the rounding of the exponent's argument gives the largest logits); measured maximum
# in DESIGN.md section 4.  A dropped P_lo . V_hi costs ~2^-13 = 1.2e-4 relative, 5x above the gate's largest value here.
ATT_C = 2.0


def relfro_gate(r):
    """[B, H]: ATT_C ((12 nblk + 4) 2^-25 + 2^-23 max|s|), the max over the sequence's valid keys"""
    smax = r["s"].abs().masked_fill(r["km"], 0.0).amax((-1, -2))
    return ATT_C * ((12 * r["nblk"][:, :, 0, 0] + 4) * 2.0 ** -25 + 2.0 ** -23 * smax)


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def S():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def lib():
    from esm_b200 import _lib
    return _lib


def make_qkv(B, T, H, seed, std=2.0):
    """fp32 [B*T, 3E] with logits of std `std` (q ~ N(0, (std/8)^2), k, v ~ N(0, 1))"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    E = 64 * H
    x = torch.randn(B * T, 3 * E, device="cuda", generator=g)
    x[:, :E] *= std / 8.0
    return x


def pad_of(B, T, lengths):
    pad = torch.zeros(B, T, dtype=torch.uint8, device="cuda")
    for b, n in enumerate(lengths):
        pad[b, n:] = 1
    return pad


def halves(x32):
    """fp32 [M, 3E] -> (qkv2 [M, 6E] fp16 hi | lo, and the hi, lo halves)"""
    hi, lo = kr.split16(x32)
    return torch.cat((hi, lo), 1).contiguous(), hi, lo


def heads(t, B, T, H, i):
    """section i (0 q, 1 k, 2 v) of [B*T, 3E] as [B, H, T, 64] float64"""
    E = 64 * H
    return t[:, i * E:(i + 1) * E].double().reshape(B, T, H, 64).transpose(1, 2)


def reference(hi, lo, pad, B, T, H):
    """float64 on hi + lo: ctx [B,H,T,64], p [B,H,T,T] (rows of an all-padding sequence 0), s, m, l = sum e^(s - m),
    the per-key relative weight error Delta (module docstring) and the number of 64-key blocks of each sequence."""
    q, k, v = (heads(hi, B, T, H, i) + heads(lo, B, T, H, i) for i in range(3))
    qh, ql, kh, kl = heads(hi, B, T, H, 0), heads(lo, B, T, H, 0), heads(hi, B, T, H, 1), heads(lo, B, T, H, 1)
    s = q @ k.transpose(-1, -2)
    keymask = torch.zeros(B, T, dtype=torch.bool, device=hi.device) if pad is None else pad.bool()
    km = keymask[:, None, None, :]
    sm = s.masked_fill(km, float("-inf"))
    m = sm.amax(-1, keepdim=True)
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    e = torch.exp(sm - m)
    l = e.sum(-1, keepdim=True)
    p = e / torch.where(l > 0, l, torch.ones_like(l))
    ctx = p @ v
    A = qh.abs() @ kh.abs().transpose(-1, -2) + ql.abs() @ kh.abs().transpose(-1, -2) + qh.abs() @ kl.abs().transpose(-1, -2)
    D = ql.abs() @ kl.abs().transpose(-1, -2)
    delta = 16 * 2.0 ** -22 * A + D + 2.0 ** -21 + 2.0 ** -23 * (s.abs() + 3 * m.abs())
    delta = delta.masked_fill(km, 0.0)
    kvlen = (~keymask).sum(-1)
    nblk = ((kvlen + 63) // 64).double()[:, None, None, None]
    return dict(q=q, k=k, v=v, s=s, m=m, l=l, p=p, ctx=ctx, delta=delta, nblk=nblk, km=km)


def ctx_bound(r):
    p, v, ctx, delta, nblk, l = r["p"], r["v"], r["ctx"], r["delta"], r["nblk"], r["l"]
    pv = p @ v.abs()
    b = (p * delta) @ v.abs() + (p * delta).sum(-1, keepdim=True) * ctx.abs()
    b = b + (12 * nblk + 4) * 2.0 ** -22 * 1.01 * pv
    b = b + 2.0 ** -21 * pv + 2.0 ** -25 * (v.abs().masked_fill(r["km"].transpose(-1, -2)[..., :1], 0.0)
                                             .sum(-2, keepdim=True) / torch.where(l > 0, l, torch.ones_like(l)))
    b = b + nblk * U * pv + (18 * nblk + 4) * U * ctx.abs()
    return b + kr.split_rep_bound(ctx)


def probs_bound(r):
    """p off by Delta_j (its own logit) + 2 max Delta (the saved maximum and row sum come from the forward kernel's
    logits) + the row sum's accumulation (18 nblk + 4) u + 1/l, the product and the fp32 store (4 u); ex2.approx
    flushes results below 2^-126 to zero"""
    p, delta, nblk = r["p"], r["delta"], r["nblk"]
    dmax = delta.amax(-1, keepdim=True)
    return p * (delta + 2 * dmax + (18 * nblk + 8) * U) + 1e-37


def run(qkv2, pad, B, T, H, probs=True):
    L = lib(); lb = L.load()
    E = 64 * H
    ctx = torch.full((B * T, 2 * E), float("nan"), dtype=torch.float16, device="cuda")
    pr = torch.full((B, H, T, T), float("nan"), device="cuda") if probs else None
    scratch = torch.empty(lb.esmb200_attention_scratch_bytes(B, T), dtype=torch.uint8, device="cuda")
    L.check(lb.esmb200_attention_split(P(qkv2), P(pad), P(ctx), P(pr), B, T, H, P(scratch), S()))
    torch.cuda.synchronize()
    return ctx, pr, scratch


def ctx_heads(ctx, B, T, H):
    E = 64 * H
    return kr.join64(ctx[:, :E], ctx[:, E:]).reshape(B, T, H, 64).transpose(1, 2)


def check(name, x32, pad, B, T, H, lengths, probs=True, stats=True):
    """Run the split kernel on split16(x32) and hold ctx, the probabilities and the saved statistics to their bounds;
    ctx bit-identical without probabilities and across two calls.  Returns the worst ratios."""
    qkv2, hi, lo = halves(x32)
    ctx, pr, scratch = run(qkv2, pad, B, T, H, probs)
    r = reference(hi, lo, pad, B, T, H)
    got = ctx_heads(ctx, B, T, H)
    assert not bool(got.isnan().any()), "ctx not written"
    live = torch.tensor([n > 0 for n in lengths], device="cuda")
    err = (got - r["ctx"]).abs()
    ratio = float((err / ctx_bound(r)).max())
    num = err.pow(2).sum((-1, -2)).sqrt()
    den = r["ctx"].pow(2).sum((-1, -2)).sqrt()
    rf = (num / den.clamp_min(1e-300))[live]                       # [live sequences, H]
    box = float((rf / relfro_gate(r)[live]).max())
    out = dict(ctx_over_bound=ratio, relfro_over_gate=box, ctx_relfro=float(rf.max()))
    for b, n in enumerate(lengths):
        if n == 0:  # an all-padding sequence: ctx exactly zero (both halves)
            assert bool((ctx[b * T:(b + 1) * T] == 0).all())
    if probs:
        assert not bool(pr.isnan().any()), "probabilities not written"
        pe = (pr.double() - r["p"]).abs()
        out["probs_over_bound"] = float((pe / probs_bound(r)).max())
        out["probs_max_abs"] = float(pe.max())
        assert bool((pr.masked_select(r["km"].expand_as(pr)) == 0).all()), "padded key columns not exactly 0"
        rows = pr.double().sum(-1)[live]
        out["rowsum_dev_over_Tu"] = float((rows - 1).abs().max()) / (T * U)
    if stats:
        mx, sm = _stats(scratch, B, T, H)
        m = r["m"][..., 0]
        dmax = r["delta"].amax(-1)
        # the saved maximum is the largest of the kernel's own logits: within the largest logit error of the row
        out["row_max_over_bound"] = float(((mx.double() - m).abs() / (dmax + 1e-30)).max())
        l_at = torch.exp(r["s"].masked_fill(r["km"], float("-inf")) - mx.double()[..., None]).sum(-1)
        lb = l_at * (dmax + (18 * r["nblk"][..., 0] + 4) * U) + 1e-30
        out["row_sum_over_bound"] = float(((sm.double() - l_at).abs() / lb).max())
        for b, n in enumerate(lengths):
            if n == 0:
                assert bool((mx[b] == 0).all()) and bool((sm[b] == 0).all())
    report(f"attention_split {name} B={B} T={T} H={H}", **out)
    assert out["ctx_over_bound"] <= 1.0 and out["relfro_over_gate"] <= 1.0, out
    for k in ("probs_over_bound", "row_max_over_bound", "row_sum_over_bound"):
        if k in out:
            assert out[k] <= 1.0, (k, out)
    if "rowsum_dev_over_Tu" in out:
        assert out["rowsum_dev_over_Tu"] <= 1.0, out
    ctx2, _, _ = run(qkv2, pad, B, T, H, probs=False)
    assert torch.equal(ctx, ctx2)  # with and without probabilities
    ctx3, _, _ = run(qkv2, pad, B, T, H, probs=False)
    assert torch.equal(ctx2, ctx3)  # two identical calls
    return out


# ---- lengths around the 64-key blocks -------------------------------------------------------------------------------
@pytest.mark.parametrize("std", [2.0, 8.0], ids=["std2", "sharp"])
@pytest.mark.parametrize("T", [1, 63, 64, 65, 127, 128, 129, 200, 1023, 1024])
def test_lengths_context_probs_and_stats(T, std):
    B, H = 3, 2
    lengths = [T, max(1, T // 2), max(1, (2 * T) // 3 - 1)]
    x = make_qkv(B, T, H, 100 + T, std)
    check(f"lengths={lengths} std={std}", x, pad_of(B, T, lengths), B, T, H, lengths)


@pytest.mark.parametrize("H", [20, 40])
def test_full_length_at_model_head_counts(H):
    """T = 1024 at the 650M (20) and 3B (40) head counts, sharp logits, one full and one ragged sequence"""
    B, T = 2, 1024
    lengths = [1024, 700]
    x = make_qkv(B, T, H, H, 8.0)
    check(f"lengths={lengths} sharp", x, pad_of(B, T, lengths), B, T, H, lengths)


def test_all_padding_sequence():
    B, T, H = 3, 300, 2
    lengths = [300, 0, 131]
    x = make_qkv(B, T, H, 7, 8.0)
    check("all padding", x, pad_of(B, T, lengths), B, T, H, lengths)


def test_left_padding_and_interior_gap_at_minus_40():
    """The first two 64-key blocks fully padded and the third partly; an interior gap across block boundaries; every
    valid logit about -40"""
    B, T, H = 2, 500, 2
    E = 64 * H
    g = torch.Generator(device="cuda").manual_seed(17)
    u = torch.randn(64, device="cuda", generator=g)
    u = u / u.norm() * (40.0 ** 0.5)
    x = 0.05 * torch.randn(B * T, 3 * E, device="cuda", generator=g)
    for h in range(H):
        x[:, h * 64:(h + 1) * 64] += u
        x[:, E + h * 64:E + (h + 1) * 64] -= u
    x[:, 2 * E:] = torch.randn(B * T, E, device="cuda", generator=g)
    pad = torch.zeros(B, T, dtype=torch.uint8, device="cuda")
    pad[0, :150] = 1
    pad[1, 40:200] = 1
    pad[1, 490:] = 1
    check("left padding, gap, logits ~-40", x, pad, B, T, H, [350, 330])


def test_running_maximum_rises_every_block():
    """Each 64-key block beats the previous maximum by ~3: every block rescales O and l"""
    B, H, T = 2, 3, 1000
    E = 64 * H
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(B * T, 3 * E, device="cuda", generator=g)
    u = torch.randn(64, device="cuda", generator=g)
    u = u / u.norm() * (8.0 ** 0.5)
    blk = (torch.arange(B * T, device="cuda").float() % T / 64).floor()
    for h in range(H):
        x[:, h * 64:(h + 1) * 64] = u + 0.1 * torch.randn(B * T, 64, device="cuda", generator=g)
        x[:, E + h * 64:E + (h + 1) * 64] = u * (0.4 * blk[:, None]) + 0.3 * torch.randn(B * T, 64, device="cuda",
                                                                                         generator=g)
    check("rising maximum", x, None, B, T, H, [T, T])


# ---- column attention -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 64, 65, 129])
@pytest.mark.parametrize("C", [1, 7])
def test_column_attention_split(R, C):
    """esmb200_column_attention_split on the row-major [B*R*C, 6E] qkv (each column a sequence of R tokens, 6E apart)
    against float64 on the column-regrouped tensor; sharp logits, ragged columns and one fully padded column (ctx
    exactly zero)."""
    L = lib(); lb = L.load()
    B, H = 2, 2
    E = 64 * H
    M = B * R * C
    g = torch.Generator(device="cuda").manual_seed(R * 10 + C)
    x = torch.randn(B, R, C, 3 * E, device="cuda", generator=g)
    x[..., :E] *= 1.0  # logits std 8
    pad = torch.zeros(B, C, R, dtype=torch.uint8, device="cuda")
    for b in range(B):
        for c in range(C):
            pad[b, c, max(1, (R * (c + 2)) // (C + 2)):] = 1 if c % 2 else 0
    pad[1, 0, :] = 1  # a column that is all padding
    qkv2, hi, lo = halves(x.reshape(M, 3 * E))
    ctx = torch.full((M, 2 * E), float("nan"), dtype=torch.float16, device="cuda")
    scratch = torch.empty(lb.esmb200_attention_scratch_bytes(B * C, R), dtype=torch.uint8, device="cuda")
    L.check(lb.esmb200_column_attention_split(P(qkv2), P(pad), P(ctx), B, R, C, H, P(scratch), S()))
    torch.cuda.synchronize()

    def regroup(t):  # [B*R*C, w] -> [B*C*R, w]
        return t.view(B, R, C, -1).permute(0, 2, 1, 3).reshape(B * C * R, -1)

    r = reference(regroup(hi), regroup(lo), pad.view(B * C, R), B * C, R, H)
    got = ctx_heads(regroup(ctx), B * C, R, H)
    assert not bool(got.isnan().any()), "ctx not written"
    ratio = float(((got - r["ctx"]).abs() / ctx_bound(r)).max())
    dead = regroup(ctx).view(B, C, R, 2 * E)[1, 0]
    assert bool((dead == 0).all()), "fully padded column not zero"
    live = (pad.view(B * C, R) == 0).any(-1)
    num = (got - r["ctx"]).pow(2).sum((-1, -2)).sqrt()[live]
    den = r["ctx"].pow(2).sum((-1, -2)).sqrt()[live]
    box = float((num / den / relfro_gate(r)[live]).max())
    report(f"attention_split column B={B} R={R} C={C} H={H}", ctx_over_bound=ratio, relfro_over_gate=box)
    assert ratio <= 1.0 and box <= 1.0
