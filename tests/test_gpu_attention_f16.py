"""GPU (-m gpu): the fp16 attention kernels against float64 softmax attention on their own fp16 q, k, v:
attention_wg_kernel (64-wide heads, 128-key blocks; esmb200_attention and esmb200_column_attention),
attention_fwd_kernel<false, 2> (128-wide heads as two 64-wide slots, 64-key blocks; esmb200_attention128) and
attention_probs_kernel<0> / <2> (the need_head_weights probabilities from the forward's saved row max and row sum).

check16 holds every call to the bounds of kernel_refs (derived there, checked against an emulation of the kernels'
arithmetic in test_kernel_refs_host.py): ctx element-wise and per (sequence, head) in rel-Frobenius norm, the
probabilities element-wise with padded key columns exactly 0 and row sums within their own bound, and the saved
statistics; an all-padding sequence gives exactly zero ctx, probabilities and statistics; ctx is
bit-identical with and without probabilities and across two calls.  Outputs are prefilled with NaN; every case prints a
PARITY line (exact checks their number of mismatching elements).  The float64
references are computed per chunk of (sequence, head) pairs, and past T = 2896 per slice of one head's query rows
(kr.attention64_rows), so that the T = 1024, 40-head cases and one head at T = 16384 stay within a few GB."""
import ctypes

import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu

CHUNK = 1 << 23  # float64 elements of one [b, h, T, T] reference tensor per chunk


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def S():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def lib():
    from esm_b200 import _lib
    return _lib


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def block_of(D):
    """keys per block of the forward kernel that runs head width D"""
    return 128 if D == 64 else 64


def pad_of(B, T, lengths):
    if lengths is None:
        return None
    pad = torch.zeros(B, T, dtype=torch.uint8, device="cuda")
    for b, n in enumerate(lengths):
        pad[b, n:] = 1
    return pad


def make_qkv(B, T, H, D, seed, std=1.0):
    """fp16 [B*T, 3 D H] with logits of std `std` (q ~ N(0, std^2 / D), k, v ~ N(0, 1))"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B * T, 3 * D * H, device="cuda", generator=g)
    x[:, :D * H] *= std / D ** 0.5
    return x.half()


def run16(qkv, pad, B, T, H, D, probs=True):
    L = lib(); lb = L.load()
    ctx = torch.full((B * T, D * H), float("nan"), dtype=torch.float16, device="cuda")
    pr = torch.full((B, H, T, T), float("nan"), device="cuda") if probs else None
    scratch = torch.empty(lb.esmb200_attention_scratch_bytes(B, T), dtype=torch.uint8, device="cuda")
    fn = lb.esmb200_attention if D == 64 else lb.esmb200_attention128
    L.check(fn(P(qkv), P(pad), P(ctx), P(pr), B, T, H, P(scratch), S()))
    torch.cuda.synchronize()
    return ctx, pr, scratch


def _heads(t, B, T, H, D, i, bs, hs):
    """section i (0 q, 1 k, 2 v; ctx: 0) of t [B*T, n D H] for sequences bs, heads hs as [b, h, T, D]"""
    E = D * H
    return t[:, i * E:(i + 1) * E].view(B, T, H, D)[bs, :, hs].transpose(1, 2)


def measure(qkv, pad, B, T, H, D, ctx, pr=None, mx=None, sm=None):
    """Worst ratios of ctx (and, when given, the probabilities and saved statistics) to their kernel_refs bounds, over
    chunks of (sequence, head) pairs; checks the exact zeros of all-padding sequences and of padded key columns."""
    padded = torch.zeros(B, T, dtype=torch.bool, device="cuda") if pad is None else pad.bool()
    dead = padded.all(-1)
    assert not bool(ctx.isnan().any()), "ctx not written"
    for b in torch.nonzero(dead).flatten().tolist():
        assert bool((ctx[b * T:(b + 1) * T] == 0).all()), "all-padding sequence: ctx not exactly 0"
    out = dict(ctx_over_bound=0.0, relfro_over_gate=0.0, ctx_relfro=0.0, ctx_absmax=0.0)
    if pr is not None:
        assert not bool(pr.isnan().any()), "probabilities not written"
        assert bool((pr.masked_select(padded[:, None, None, :].expand_as(pr)) == 0).all()), "padded key column not 0"
        assert bool((pr[dead] == 0).all()), "all-padding sequence: probabilities not exactly 0"
        out.update(probs_over_bound=0.0, rowsum_over_bound=0.0, row_max_over_bound=0.0, row_sum_over_bound=0.0)
    if mx is not None:
        assert bool((mx[dead] == 0).all()) and bool((sm[dead] == 0).all()), "all-padding sequence: statistics not 0"
    nb = max(1, min(B, CHUNK // (T * T)))
    nh = max(1, min(H, CHUNK // (nb * T * T)))
    for b0 in range(0, B, nb):
        bs = slice(b0, min(B, b0 + nb))
        live = ~dead[bs]
        for h0 in range(0, H, nh):
            hs = slice(h0, min(H, h0 + nh))
            q, k, v = (_heads(qkv, B, T, H, D, i, bs, hs) for i in range(3))
            err2 = 0.0
            terms = [0.0, 0.0, 0.0]
            for i0, r in kr.attention64_rows(q, k, v, padded[bs], block_of(D), CHUNK):
                rows = slice(i0, i0 + r["q"].shape[-2])
                err = _heads(ctx, B, T, H, D, 0, bs, hs)[:, :, rows].double() - r["ctx"]
                out["ctx_over_bound"] = max(out["ctx_over_bound"], float((err.abs() / kr.attn_ctx_bound(r)).max()))
                err2 = err2 + err.pow(2).sum((-1, -2))
                terms = [a + t for a, t in zip(terms, kr.attn_relfro_terms(r))]
                out["ctx_absmax"] = max(out["ctx_absmax"], float(r["ctx"].abs().max()))
                if pr is not None:
                    pb = kr.attn_probs_bound(r)
                    prow = pr[bs, hs, rows].double()
                    out["probs_over_bound"] = max(out["probs_over_bound"], float(((prow - r["p"]).abs() / pb).max()))
                    dev = (prow.sum(-1) - 1).abs()[live]
                    out["rowsum_over_bound"] = max(out["rowsum_over_bound"],
                                                   float((dev / kr.attn_rowsum_bound(r)[live]).max()))
                if mx is not None:
                    m, s = mx[bs, hs, rows].double(), sm[bs, hs, rows].double()
                    out["row_max_over_bound"] = max(out["row_max_over_bound"],
                                                    float(((m - r["m"][..., 0]).abs() / kr.attn_max_bound(r)).max()))
                    l_at = torch.exp(r["s"].masked_fill(r["km"], float("-inf")) - m[..., None]).sum(-1)
                    out["row_sum_over_bound"] = max(out["row_sum_over_bound"],
                                                    float(((s - l_at).abs() / kr.attn_sum_bound(r, l_at)).max()))
                del r
            rf = err2.sqrt() / terms[2].sqrt().clamp_min(1e-300)
            if bool(live.any()):
                gate = kr.attn_relfro_combine(*terms)
                out["relfro_over_gate"] = max(out["relfro_over_gate"], float((rf / gate)[live].max()))
                out["ctx_relfro"] = max(out["ctx_relfro"], float(rf[live].max()))
    return out


def exact(name, got, want):
    """PARITY line of an exact check: the number of elements of `got` that differ from `want` (bit patterns)"""
    bad = int((got.view(torch.int16) != want.view(torch.int16)).sum()) if got.dtype == torch.float16 else \
        int((got != want).sum())
    report(name, mismatches=float(bad))
    return bad == 0 and torch.equal(got, want)


def assert_within(name, out):
    report(name, **out)
    for k, x in out.items():
        if k.endswith("_bound") or k.endswith("_gate"):
            assert x <= 1.0, (k, out)


def check16(name, qkv, pad, B, T, H, D, probs=True):
    """Run the fp16 attention (esmb200_attention, or esmb200_attention128 at D = 128) and hold it to the bounds; ctx
    bit-identical without probabilities and across two calls.  Returns the worst ratios."""
    from test_gpu_attention_wg import _stats
    ctx, pr, scratch = run16(qkv, pad, B, T, H, D, probs)
    mx, sm = _stats(scratch, B, T, H) if probs else (None, None)
    out = measure(qkv, pad, B, T, H, D, ctx, pr, mx, sm)
    assert_within(f"attention_f16 D={D} {name} B={B} T={T} H={H}", out)
    ctx2, _, _ = run16(qkv, pad, B, T, H, D, probs=False)
    assert torch.equal(ctx, ctx2)  # with and without probabilities
    ctx3, _, _ = run16(qkv, pad, B, T, H, D, probs=False)
    assert torch.equal(ctx2, ctx3)  # two identical calls
    return out


def run_column(qkv, pad, B, R, C, H):
    """esmb200_column_attention on the row-major [B*R*C, 3E] qkv, pad [B, C, R]; returns ctx [B*R*C, E]"""
    L = lib(); lb = L.load()
    E = 64 * H
    ctx = torch.full((B * R * C, E), float("nan"), dtype=torch.float16, device="cuda")
    scratch = torch.empty(lb.esmb200_attention_scratch_bytes(B * C, R), dtype=torch.uint8, device="cuda")
    L.check(lb.esmb200_column_attention(P(qkv), P(pad), P(ctx), B, R, C, H, P(scratch), S()))
    torch.cuda.synchronize()
    return ctx


def check_column(name, qkv, pad, B, R, C, H):
    """Column attention against float64 on the column-regrouped tensor [B*C*R, 3E]; bit-identical across two calls"""
    ctx = run_column(qkv, pad, B, R, C, H)

    def regroup(t):  # [B*R*C, w] -> [B*C*R, w]
        return t.view(B, R, C, -1).permute(0, 2, 1, 3).reshape(B * C * R, -1)

    out = measure(regroup(qkv), None if pad is None else pad.view(B * C, R), B * C, R, H, 64, regroup(ctx))
    assert_within(f"attention_f16 column {name} B={B} R={R} C={C} H={H}", out)
    assert torch.equal(ctx, run_column(qkv, pad, B, R, C, H))
    return out, ctx


# ---- lengths around the key blocks of both kernels ------------------------------------------------------------------
T_SWEEP = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 1023, 1024]


@pytest.mark.parametrize("std", [1.0, 8.0], ids=["diffuse", "sharp"])
@pytest.mark.parametrize("T", T_SWEEP)
@pytest.mark.parametrize("D", [64, 128])
def test_lengths_at_block_edges(D, T, std):
    B, H = 3, 2
    lengths = [T, max(1, T // 2), max(1, (2 * T) // 3 - 1)]
    qkv = make_qkv(B, T, H, D, 1000 * D + T + int(std), std)
    check16(f"lengths={lengths} std={std}", qkv, pad_of(B, T, lengths), B, T, H, D)


@pytest.mark.parametrize("D,B,H", [(64, 4, 20), (64, 4, 40), (128, 2, 40)])
def test_full_length_at_model_head_counts(D, B, H):
    """T = 1024 at the 650M (20 heads) and 3B (40) head counts, four sequences so that each persistent CTA of the wg
    kernel walks several items; the 15B shape (40 heads of 128, 8 query tiles) on the two-slot kernel"""
    T = 1024
    lengths = [1024, 1000, 700, 513][:B]
    qkv = make_qkv(B, T, H, D, 7 * H + D, 1.0)
    check16(f"lengths={lengths}", qkv, pad_of(B, T, lengths), B, T, H, D)


def test_all_padding_sequence_d128():
    B, T, H = 3, 300, 2
    lengths = [300, 0, 131]
    check16("all padding", make_qkv(B, T, H, 128, 7, 8.0), pad_of(B, T, lengths), B, T, H, 128)


def rising_qkv(B, T, H, D, seed, rise_every=64):
    """Each `rise_every`-key block beats the previous maximum by ~3.2: every block rescales O and l"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    E = D * H
    x = torch.randn(B * T, 3 * E, device="cuda", generator=g)
    u = torch.randn(D, device="cuda", generator=g)
    u = u / u.norm() * (8.0 ** 0.5)
    blk = (torch.arange(B * T, device="cuda") % T // rise_every).float()
    for h in range(H):
        x[:, h * D:(h + 1) * D] = u + 0.1 * torch.randn(B * T, D, device="cuda", generator=g)
        x[:, E + h * D:E + (h + 1) * D] = u * (0.4 * blk[:, None]) + 0.3 * torch.randn(B * T, D, device="cuda",
                                                                                       generator=g)
    return x.half()


@pytest.mark.parametrize("D", [64, 128])
def test_running_maximum_rises_every_64_keys(D):
    """The rise per 64-key block: every block of the two-slot kernel and both halves of every wg block"""
    B, H, T = 2, 3, 1000
    check16("rising maximum per 64 keys", rising_qkv(B, T, H, D, 5), None, B, T, H, D)


# ---- neighbour isolation --------------------------------------------------------------------------------------------
POISON_V = 1e3


def poisoned_qkv(n, T, H, D, seed, pad=None, lead=True):
    """(fp16 [n*T, 3E], e): every query along the unit direction e (logits of std ~2 against ordinary keys), and keys
    15 e that score +30 against every query at the padded rows and (lead) at the rows a sequence's last key box reads
    past its end: the first lead_rows(T) rows of the next sequence.  Their values are +1e3 in even sequences and -1e3
    in odd ones, so a leaked key moves ctx by ~1e3 even in a sequence whose own valid keys are poisoned."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    E = D * H
    x = torch.randn(n, T, 3, H, D, device="cuda", generator=g)
    e = torch.randn(D, device="cuda", generator=g)
    e = e / e.norm()
    x[:, :, 0] = 2.0 * e + 0.5 / D ** 0.5 * x[:, :, 0]
    poison = torch.zeros(n, T, dtype=torch.bool, device="cuda")
    if lead:
        poison[1:, :lead_rows(T)] = True
    if pad is not None:
        poison |= pad.bool()
    sign = (1 - 2 * (torch.arange(n, device="cuda") % 2)).float()[:, None].expand(n, T)
    x[:, :, 1][poison] = 15.0 * e
    x[:, :, 2][poison] = POISON_V * sign[poison][:, None, None]
    return x.reshape(n * T, 3 * E).half(), e


def lead_rows(T):
    """rows of the next sequence that a sequence of T tokens reads in its last 128-key box (64-key boxes read fewer)"""
    return min(T, (T + 127) // 128 * 128 - T)


@pytest.mark.parametrize("masked", [False, True], ids=["no_mask", "mask"])
@pytest.mark.parametrize("T", [100, 200, 333])
@pytest.mark.parametrize("D", [64, 128])
def test_neighbour_rows_do_not_leak(D, T, masked):
    """T not a multiple of either key block: the last key box of each sequence reads the next sequence's first rows
    (the last sequence's box runs past the tensor), which score +30 against this sequence's queries with values of
    +-1e3.  Without a mask those rows are valid keys of their own sequence; with a mask they are padded there, as are
    each ragged sequence's tail rows (poisoned too), so that no sequence has a poisoned valid key and every ctx stays
    O(1).  Any key counted past T, or a padded one, moves ctx by ~1e3."""
    check_neighbour_isolation(D, T, masked)


def check_neighbour_isolation(D, T, masked):
    """test_neighbour_rows_do_not_leak at any T"""
    B, H = 3, 2
    pad = None
    if masked:
        pad = pad_of(B, T, [T, T - 37, T // 3])
        pad[1:, :lead_rows(T)] = 1
    qkv, _ = poisoned_qkv(B, T, H, D, T + D, pad)
    out = check16("neighbour isolation " + ("mask" if masked else "no mask"), qkv, pad, B, T, H, D)
    ctx, _, _ = run16(qkv, pad, B, T, H, D, probs=False)
    clean = ctx if masked else ctx[:T]  # without a mask only sequence 0 has no poisoned valid key
    assert float(clean.float().abs().max()) < 20.0
    assert out["ctx_relfro"] < 2e-3


@pytest.mark.parametrize("masked", [False, True], ids=["no_mask", "mask"])
@pytest.mark.parametrize("R", [65, 200])
def test_column_neighbour_rows_do_not_leak(R, masked):
    """Column attention, C = 7: the rows past R of a column's last key box belong to the next alignment's first rows
    (same column), poisoned as above; with a mask they are padded in their own alignment, and each column's padded
    tail rows are poisoned too, so that no column has a poisoned valid key"""
    B, C, H = 2, 7, 2
    E = 64 * H
    nlead = lead_rows(R)
    pad = None
    if masked:
        pad = torch.zeros(B, C, R, dtype=torch.uint8, device="cuda")
        for c in range(C):
            pad[:, c, R - 1 - 9 * c:] = 1
        pad[1:, :, :nlead] = 1
    x, e = poisoned_qkv(B * C, R, H, 64, R + 3, None if pad is None else pad.view(B * C, R), lead=False)
    # column sequences [B, C, R] -> row-major [B, R, C]: the rows past R of alignment b are alignment b + 1's first rows
    qkv = x.view(B, C, R, 3 * E).permute(0, 2, 1, 3).contiguous().view(B * R * C, 3 * E)
    lead = torch.zeros(B, R, C, dtype=torch.bool, device="cuda")
    lead[1:, :nlead] = True
    y = qkv.view(B, R, C, 3, H, 64)
    y[:, :, :, 1][lead] = (15.0 * e).half()
    y[:, :, :, 2][lead] = POISON_V
    _, ctx = check_column(f"neighbour isolation {'mask' if masked else 'no mask'}", qkv, pad, B, R, C, H)
    clean = ctx if masked else ctx.view(B, R * C, E)[0]  # without a mask alignment 1's first rows are valid poison
    assert float(clean.float().abs().max()) < 20.0


# ---- one-hot rows at D = 128 ----------------------------------------------------------------------------------------
def test_one_hot_rows_read_every_value_exactly_d128():
    """Query i scores 60 on key perm[i] and at most ~25 on every other key, so its fp16 P row is exactly one-hot and
    ctx row i is v[perm[i]] bit for bit in all 128 columns: pins both slots of V and O over every 64-key block."""
    B, T, H, D = 1, 384, 1, 128
    g = torch.Generator(device="cpu").manual_seed(3)
    perm = torch.randperm(T, generator=g)
    k = torch.randn(T, D, generator=g)
    k = k / k.norm(dim=1, keepdim=True) * D ** 0.5  # |k|^2 = 128; k_i . k_j ~ N(0, 128) for i != j
    qkv = torch.empty(T, 3 * D)
    qkv[:, :D] = k[perm] * (60.0 / D)
    qkv[:, D:2 * D] = k
    qkv[:, 2 * D:] = torch.randn(T, D, generator=g)
    qkv = qkv.half().cuda()
    s = qkv[:, :D].float() @ qkv[:, D:2 * D].float().t()
    top2 = s.topk(2, dim=1).values
    assert float((top2[:, 0] - top2[:, 1]).min()) > 25.0  # exp(-25) is below the smallest fp16 subnormal
    ctx, _, _ = run16(qkv, None, B, T, H, D, probs=False)
    assert exact(f"attention_f16 D={D} one-hot rows B={B} T={T} H={H}", ctx, qkv[perm.cuda(), 2 * D:])


# ---- column attention -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 7])
@pytest.mark.parametrize("R", [1, 64, 65, 127, 128, 129, 1024])
def test_column_attention_at_block_edges(R, C):
    """MSA-1b's 12 heads; ragged columns and one fully padded column, whose ctx is exactly zero"""
    B, H = 2, 12
    E = 64 * H
    g = torch.Generator(device="cuda").manual_seed(R * 10 + C)
    qkv = torch.randn(B * R * C, 3 * E, device="cuda", generator=g)
    qkv[:, :E] *= 1.0 / 8.0
    qkv = qkv.half()
    pad = torch.zeros(B, C, R, dtype=torch.uint8, device="cuda")
    for b in range(B):
        for c in range(C):
            pad[b, c, max(1, (R * (c + 2)) // (C + 2)):] = 1 if c % 2 else 0
    pad[1, 0, :] = 1  # a column that is all padding
    _, ctx = check_column("ragged, one dead column", qkv, pad, B, R, C, H)
    assert bool((ctx.view(B, R, C, E)[1, :, 0] == 0).all())
