"""GPU (-m gpu): the MSA Transformer's tied row attention (esmb200_tied_row_attention and _split: tied_scores_kernel,
tied_softmax_kernel and tied_pv_kernel, <false> fp16 and <true> fp32x3) against float64 on the kernels' own operands.

check_tied runs each case twice.  The call without probabilities leaves the kernels' intermediates in scratch: the
fp32 logits S [H,B,C,C] and P [H*B*C, Cp] (fp32x3: [H*B*C, 2 Cp], hi | lo).  Each stage is then held to its own
kernel_refs bound on its own actual inputs (logits on q, k; P on softmax of the kernel's S; ctx on the kernel's P V),
which stays tight at every R, and ctx end to end to tied64 (element-wise and per (alignment, head) in rel-Frobenius
norm; loose for fp16 at large R, where the stage bounds do the detecting).  The call with probabilities checks them
and their row sums, and that P and ctx are the same bits.  Exact checks: every output written (outputs and scratch
prefilled with NaN), P exactly 0 in columns [C, Cp), probabilities exactly 0 at padded key columns (uniform 1/C when
an alignment's keys are all padded), and with fp32x3 |lo| within half an fp16 ulp of hi.  Every case prints a PARITY
line with its worst ratios.

The cases walk the kernels' edges: the scores kernel's 128 x 128 tiles and its 4-stage (fp32x3: 3-stage) ring over
the alignment rows R, the softmax's one warp per row up to C = 1024, and the P V kernel's 128 query columns x 4
alignment rows per CTA with 64-key tiles in a 2-stage ring.  Boxes that overhang C read into the next alignment row;
the isolation case checks that nothing read there reaches a result."""
import ctypes

import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu

PRECISIONS = pytest.mark.parametrize("split", [False, True], ids=["fp16", "fp32x3"])


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def S():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def lib():
    from esm_b200 import _lib
    return _lib


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def entry(split):
    lb = lib().load()
    if split:
        return lb.esmb200_tied_row_attention_split, lb.esmb200_tied_row_attention_split_scratch_bytes
    return lb.esmb200_tied_row_attention, lb.esmb200_tied_row_attention_scratch_bytes


def make_qkv(B, R, C, H, seed, std=3.0, split=False, key_pad=None, zero_q=True):
    """qkv [B*R*C, 3E] fp16 (fp32x3: [B*R*C, 6E], hi | lo of fp32 draws) with summed logits of std `std`; q is zeroed at
    padded key columns (as the MSA stack does) unless zero_q is False"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(B, R, C, 3, H, 64, device="cuda", generator=g)
    x[:, :, :, 0] *= std / (64 * R) ** 0.5
    if key_pad is not None and zero_q:
        x[:, :, :, 0] *= (~key_pad.bool())[:, None, :, None, None]
    return pack(x, split)


def pack(x, split):
    """[B,R,C,3,H,64] fp32 -> the kernel's qkv"""
    x = x.reshape(-1, x.shape[3] * x.shape[4] * 64)
    return torch.cat(kr.split16(x), 1).contiguous() if split else x.half()


def scratch_views(scratch, B, C, H, split):
    """(S [H,B,C,C] fp32, P [H*B*C, Cp] fp16 or [H*B*C, 2 Cp] hi | lo) inside the scratch of a call without
    probabilities: the logits at the scratch base rounded up to 1024 bytes, P 1024-aligned after them (api.cu
    tied_row_impl / tied_scratch_bytes).  A changed layout fails here rather than reading garbage."""
    Cp, pf = (C + 63) // 64 * 64, 2 if split else 1
    up = lambda n: (n + 1023) // 1024 * 1024  # noqa: E731
    s_bytes, p_bytes = H * B * C * C * 4, H * B * C * Cp * 2 * pf
    assert entry(split)[1](B, C, H) == up(s_bytes) + up(p_bytes) + 2048, "tied scratch layout changed"
    base = (-scratch.data_ptr()) % 1024
    Sv = scratch[base:base + s_bytes].view(torch.float32).view(H, B, C, C)
    Pv = scratch[base + up(s_bytes):base + up(s_bytes) + p_bytes].view(torch.float16).view(H * B * C, pf * Cp)
    return Sv, Pv


def run_tied(qkv, key_pad, B, R, C, H, split, probs):
    """one call on NaN-prefilled outputs and 0xFF-prefilled scratch -> (ctx, probabilities or None, S, P)"""
    L = lib()
    fn, nbytes_of = entry(split)
    nbytes = nbytes_of(B, C, H)
    scratch = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")
    ctx = torch.full((B * R * C, (2 if split else 1) * 64 * H), float("nan"), dtype=torch.float16, device="cuda")
    pr = torch.full((H, B, C, C), float("nan"), device="cuda") if probs else None
    L.check(fn(P(qkv), P(key_pad), P(ctx), P(pr), B, R, C, H, P(scratch), nbytes, S()))
    torch.cuda.synchronize()
    Sv, Pv = scratch_views(scratch, B, C, H, split)
    return ctx, pr, Sv.clone(), Pv.clone()


def joined(ctx, B, R, C, H, split):
    """ctx as float64 [B,R,C,H,64] (hi + lo with fp32x3)"""
    E = 64 * H
    if split:
        return kr.join64(ctx[:, :E], ctx[:, E:]).view(B, R, C, H, 64)
    return ctx.double().view(B, R, C, H, 64)


def same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def lo_within_half_ulp(hi, lo):
    h = hi.double()
    half = torch.where(h == 0, torch.full_like(h, kr.F16_HALF_QUANTUM), kr.half_ulp16(h))
    return bool((lo.double().abs() <= half).all())


def _ratio(err, bound):
    return float((err.abs() / bound.clamp_min(1e-300)).max())


def check_tied(name, qkv, key_pad, B, R, C, H, split):
    """Both calls of one case, every check above; returns (ctx of the call without probabilities, probabilities)."""
    Cp, E = (C + 63) // 64 * 64, 64 * H
    prec = "fp32x3" if split else "fp16"
    ctx_a, _, S_a, P_a = run_tied(qkv, key_pad, B, R, C, H, split, probs=False)
    ctx_b, pr, _, P_b = run_tied(qkv, key_pad, B, R, C, H, split, probs=True)
    # exact checks
    assert not bool(ctx_a.isnan().any()) and not bool(pr.isnan().any()), "output not written"
    assert not bool(S_a.isnan().any()) and not bool(P_a.isnan().any()), "scratch logits / P not written"
    assert same_bits(ctx_a, ctx_b) and same_bits(P_a, P_b), "with and without probabilities differ"
    Ph = P_a.view(H, B, C, -1).double()
    halves = Ph.view(H, B, C, 2 if split else 1, Cp)
    assert bool((halves[..., C:] == 0).all()), "P not exactly 0 in columns [C, Cp)"
    km = kr.tied_pad(key_pad, B, C, qkv.device).expand(H, B, C, C)
    dead = km.all(-1, keepdim=True).expand_as(km)
    uniform = torch.ones((), device="cuda") / C
    assert bool((pr[km & ~dead] == 0).all()), "probability at a padded key column not exactly 0"
    assert bool((pr[dead] == uniform).all()), "all keys padded: probabilities not uniform 1/C"
    if split:
        assert lo_within_half_ulp(P_a[:, :Cp], P_a[:, Cp:]), "P lo outside half an ulp of hi"
        assert lo_within_half_ulp(ctx_a[:, :E], ctx_a[:, E:]), "ctx lo outside half an ulp of hi"
    # stage bounds on the kernels' own inputs
    r = kr.tied64(qkv, key_pad, B, R, C, H, split)
    out = dict(logits=_ratio(S_a.double() - r["s"], r["lerr"]))
    sr = kr.tied_softmax64(S_a, key_pad)
    p_hi = halves[..., 0, :C]
    p_lo = halves[..., 1, :C] if split else None
    p_val = p_hi if p_lo is None else p_hi + p_lo
    out["P"] = _ratio(p_val - sr["p"], kr.tied_P_bound(sr, split))
    out["probs"] = _ratio(pr.double() - sr["p"], kr.tied_probs_bound(sr))
    out["rowsum"] = float((pr.double().sum(-1) - 1).abs().max()) / kr.tied_rowsum_bound(C)
    _, hi, lo = kr.tied_operands(qkv, B, R, C, H, split)
    pv_ref, pv_b = kr.tied_pv(p_hi, p_lo, hi[:, :, :, 2], None if lo is None else lo[:, :, :, 2], Cp)
    got = joined(ctx_a, B, R, C, H, split)
    out["pv"] = _ratio(got - pv_ref, pv_b)
    del pv_ref, pv_b, hi, lo
    # end to end
    out["ctx"] = _ratio(got - r["ctx"], kr.tied_ctx_bound(r))
    rf = (got - r["ctx"]).pow(2).sum((1, 2, 4)).sqrt() / r["ctx"].pow(2).sum((1, 2, 4)).sqrt().clamp_min(1e-300)
    out["gate"] = float((rf / kr.tied_relfro_gate(r)).max())
    out["ctx_relfro"] = float(rf.max())
    report(f"tied_row {prec} {name} (B,R,C,H)=({B},{R},{C},{H})", **{
        (k if k == "ctx_relfro" else k + "_over_bound"): v for k, v in out.items()})
    bad = {k: v for k, v in out.items() if k != "ctx_relfro" and not v <= 1.0}
    assert not bad, f"{name}: over the bound: {bad}"
    return ctx_a, pr


def per_alignment_pad(B, C):
    """[B,C] uint8: alignment 0 pads its trailing C // 7 columns, alignment 1 column C // 3, the rest nothing"""
    pad = torch.zeros(B, C, dtype=torch.uint8, device="cuda")
    pad[0, C - C // 7:] = 1
    if B > 1 and C >= 3:
        pad[1, C // 3] = 1
    return pad


# ---- sweeps over the tiles and rings --------------------------------------------------------------------------------
C_SWEEP = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 511, 513, 1023, 1024]
R_SWEEP = [1, 2, 3, 4, 5, 7, 8, 9, 63, 64, 65, 256, 1024]


@PRECISIONS
@pytest.mark.parametrize("R", [1, 5])
@pytest.mark.parametrize("C", C_SWEEP)
def test_tied_c_sweep(C, R, split):
    B, H = 2, 2
    pad = per_alignment_pad(B, C)
    check_tied("C sweep", make_qkv(B, R, C, H, seed=C * 10 + R, split=split, key_pad=pad), pad, B, R, C, H, split)


@PRECISIONS
@pytest.mark.parametrize("C", [65, 129])
@pytest.mark.parametrize("R", R_SWEEP)
def test_tied_r_sweep(R, C, split):
    B, H = 2, 1
    pad = per_alignment_pad(B, C)
    check_tied("R sweep", make_qkv(B, R, C, H, seed=R * 10 + C, split=split, key_pad=pad), pad, B, R, C, H, split)


@PRECISIONS
@pytest.mark.parametrize("B,R,C,H", [(2, 64, 256, 12), (1, 16, 1024, 2), (1, 1024, 16, 2), (13107, 1, 2, 5)],
                         ids=["msa1b", "16k-tokens-wide", "16k-tokens-deep", "BH-65535"])
def test_tied_model_and_limit_shapes(B, R, C, H, split):
    pad = per_alignment_pad(B, C)
    check_tied("shape", make_qkv(B, R, C, H, seed=B + R + C, split=split, key_pad=pad), pad, B, R, C, H, split)


@PRECISIONS
@pytest.mark.parametrize("std", [1.0, 3.0, 8.0])
def test_tied_logit_scales(std, split):
    B, R, C, H = 2, 5, 257, 2
    pad = per_alignment_pad(B, C)
    check_tied(f"logit std {std}", make_qkv(B, R, C, H, seed=int(std), std=std, split=split, key_pad=pad), pad,
               B, R, C, H, split)


def sylvester(n):
    h = torch.ones(1, 1)
    while h.shape[0] < n:
        h = torch.cat([torch.cat([h, h], 1), torch.cat([h, -h], 1)], 0)
    return h


@PRECISIONS
@pytest.mark.parametrize("C", [100, 128])
def test_tied_one_hot_rows(C, split):
    """Keys carry distinct +-1 Hadamard codes and query i the code of key pi(i), scaled by 0.5, in every alignment
    row: the logits are 32 R at key pi(i) and 0 or -32 R elsewhere, so P is exactly one-hot, ctx is the selected V
    row, bit for bit, and the fp32 probabilities are exactly 1 at pi(i) and below 2^-126 elsewhere."""
    B, R, H = 2, 3, 2
    codes = torch.cat([sylvester(64), -sylvester(64)])  # [128, 64]
    g = torch.Generator().manual_seed(C)
    x = torch.randn(B, R, C, 3, H, 64, generator=g)
    pick = torch.stack([torch.randperm(C, generator=g) for _ in range(B * H)]).view(B, H, C)
    for b in range(B):
        for h in range(H):
            x[b, :, :, 1, h] = codes[:C]
            x[b, :, :, 0, h] = 0.5 * codes[pick[b, h]]
    onehot = torch.zeros(H, B, C, C)
    onehot.scatter_(-1, pick.permute(1, 0, 2).contiguous()[..., None], 1.0)
    qkv = pack(x.cuda(), split)
    ctx, pr = check_tied("one-hot", qkv, None, B, R, C, H, split)
    _, hi, lo = kr.tied_operands(qkv, B, R, C, H, split)
    v = hi[:, :, :, 2] if lo is None else hi[:, :, :, 2] + lo[:, :, :, 2]  # [B,R,C,H,64]
    want = kr._pv(onehot.cuda().double(), v)  # exact: one product by 1, the rest by 0
    got = joined(ctx, B, R, C, H, split)
    prc = pr.cpu()  # ex2.approx keeps e^-96 as an fp32 subnormal: the other probabilities are below 2^-126, not 0
    bad_ctx = int((got != want).sum())
    bad_p = int((prc[onehot == 1] != 1).sum()) + int((prc[onehot == 0] >= 2.0 ** -126).sum())
    report(f"tied_row {'fp32x3' if split else 'fp16'} one-hot exact C={C}", ctx_mismatches=float(bad_ctx),
           probs_mismatches=float(bad_p))
    bad = bad_ctx + bad_p
    assert bad == 0


# ---- key padding ----------------------------------------------------------------------------------------------------
def padding_case(kind, B, C):
    if kind == "none":
        return None
    pad = torch.zeros(B, C, dtype=torch.uint8, device="cuda")
    if kind == "trailing":
        pad[:, C - 40:] = 1
    elif kind == "interior":
        pad[:, [10, 64, 127, 128, 200]] = 1
        pad[:, 100:111] = 1
    elif kind == "one-alignment-all":
        pad[1] = 1
    elif kind in ("per-alignment", "q-not-zeroed"):
        pad[0, C - 40:] = 1
        pad[2, 17] = 1
        pad[2, C - 100:] = 1
    return pad


@PRECISIONS
@pytest.mark.parametrize("kind", ["none", "trailing", "interior", "one-alignment-all", "per-alignment",
                                  "q-not-zeroed"])
def test_tied_key_padding(kind, split):
    """The entry point reads key_pad [B,C] at stride C.  It does not zero q (the stack does): "q-not-zeroed" keeps q
    at the padded columns, whose logits are then computed and replaced by -10000."""
    B, R, C, H = 3, 6, 300, 2
    pad = padding_case(kind, B, C)
    qkv = make_qkv(B, R, C, H, seed=len(kind), split=split, key_pad=pad, zero_q=kind != "q-not-zeroed")
    check_tied(f"key_pad {kind}", qkv, pad, B, R, C, H, split)


@PRECISIONS
@pytest.mark.parametrize("C", [65, 100, 129])
def test_tied_alignments_are_isolated(C, split):
    """Alignments 0 and 2 replaced by keys scoring about +30 against alignment 1's queries and values of +-6e4:
    alignment 1's ctx and probabilities are bit-identical to the unperturbed run and to alignment 1 run alone.  With
    C % 128 and C % 64 != 0 the scores and P V boxes overhang into the next alignment row."""
    B, R, H = 3, 5, 2
    pad = per_alignment_pad(B, C)
    pad[1, C - 7:] = 1
    g = torch.Generator(device="cuda").manual_seed(C)
    x = torch.randn(B, R, C, 3, H, 64, device="cuda", generator=g)
    x[:, :, :, 0] *= 3.0 / (64 * R) ** 0.5
    x[:, :, :, 0] *= (~pad.bool())[:, None, :, None, None]
    u = x[1, :, :, 0].mean(1)                                    # [R,H,64]: alignment 1's mean query per row
    alpha = 30.0 / u.pow(2).sum((0, 2))                          # [H]
    xp = x.clone()
    for b in (0, 2):
        xp[b, :, :, 1] = (alpha[None, :, None] * u)[:, None]
        xp[b, :, :, 2] = 6e4 * torch.sign(torch.randn(R, C, H, 64, device="cuda", generator=g))
    rows = slice(R * C, 2 * R * C)
    runs = []
    for y, bb in ((x, B), (xp, B), (x[1:2], 1)):
        kp = pad if bb == B else pad[1:2].contiguous()
        ctx, pr, _, _ = run_tied(pack(y, split), kp, bb, R, C, H, split, probs=True)
        runs.append((ctx[rows] if bb == B else ctx, pr[:, 1] if bb == B else pr[:, 0]))
    bad = sum(int((a.view(torch.int16) != runs[0][0].view(torch.int16)).sum()) + int((p != runs[0][1]).sum())
              for a, p in runs[1:])
    report(f"tied_row {'fp32x3' if split else 'fp16'} isolation C={C}", mismatches=float(bad))
    assert bad == 0
    check_tied("isolation perturbed", pack(xp, split), pad, B, R, C, H, split)


# ---- refusals, with real buffers; tests/test_msa_host.py checks them without a device ------------------------------
@PRECISIONS
@pytest.mark.parametrize("case", ["C=1025", "BH=65536", "H=65", "scratch-short", "null-qkv", "null-ctx",
                                  "null-scratch"])
def test_tied_refusals_launch_nothing(case, split):
    L = lib(); lb = L.load()
    B, R, C, H = {"C=1025": (1, 1, 1025, 1), "BH=65536": (1024, 1, 1, 64), "H=65": (1, 1, 1, 65)}.get(case, (1, 2, 3, 1))
    fn, nbytes_of = entry(split)
    pf = 2 if split else 1
    nbytes = nbytes_of(B, C, H)
    qkv = torch.zeros(B * R * C, pf * 3 * 64 * H, dtype=torch.float16, device="cuda")
    ctx = torch.full((B * R * C, pf * 64 * H), float("nan"), dtype=torch.float16, device="cuda")
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    args = [P(qkv), None, P(ctx), None, B, R, C, H, P(scratch), nbytes - (case == "scratch-short"), S()]
    if case.startswith("null"):
        args[{"null-qkv": 0, "null-ctx": 2, "null-scratch": 8}[case]] = None
    torch.cuda.synchronize()
    before = lb.esmb200_launch_count()
    rc = fn(*args)
    err = lb.esmb200_last_error().decode()
    torch.cuda.synchronize()
    want = {"C=1025": (-1, "1024"), "scratch-short": (-4, "scratch too small")}.get(
        case, (-1, "null argument" if case.startswith("null") else "bad shape"))
    assert (rc, want[1] in err) == (want[0], True), (rc, err)
    assert lb.esmb200_launch_count() == before and bool(ctx.isnan().all())
