"""GPU (-m gpu): the three embedding prologues against float64 (kernel_refs.embed_esm2_64 / embed_esm1b_64 /
embed_msa_64), at the edges of their launch grids and register tilings.

  * embed_tokens_kernel (ESM-2): the chunked grid (chunks = min(ceil(8 n_sms / B), ceil(T / 4))) at B = 1, one chunk,
    T < 4 and trailing empty chunks; <mask> tokens that lie only outside most blocks' own chunk; left, interior and
    whole-sequence pads; every non-pad token a <mask>; E from 4 to 5120.  Without token_dropout the gather is exact;
    with it the result is within the scale's roundings of float64 and bit-identical to the reference's three fp32 ops.
  * esm1b_embed_kernel<4 | 10 | 20>: positions carried across 32-token ballots and chunk boundaries with pads exactly
    on them, T = 1 .. 1026, LayerNorm and token_dropout on and off, another padding index, and the longest sequence
    (T = 12288) at a batch large enough for one chunk per sequence.
  * msa_embed_kernel<4 | 10 | 20>: C across the ballot edges up to 1024 and at the limit 12288, R up to 130 with two
    alignments (msa_pos has more rows than R, so a wrong row index reads another row), msa_pos absent, E wide and 1
    wide, leading / interior / whole-row / whole-column pads, and tables with a large common offset.

Every output buffer starts as NaN.  Argument errors return -1 and launch nothing."""
import pytest
import torch

import kernel_refs as kr

pytestmark = pytest.mark.gpu

PAD, MASK = 1, 32


def _lib():
    from esm_b200 import _lib
    return _lib


def S():
    return torch.cuda.current_stream().cuda_stream


def P(t):
    return t.data_ptr() if t is not None else None


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def same_bits(a, b):
    """torch.equal with NaN equal to NaN"""
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(nan=0.0), b.nan_to_num(nan=0.0))


def worst(err, bound):
    """max of err / bound over the finite entries of bound's reference (NaN positions are compared separately)"""
    ok = err.isfinite()
    return float((err[ok] / bound[ok]).max()) if bool(ok.any()) else 0.0


def sequence_tokens(B, T, seed, pad=PAD, mask=MASK, marks=()):
    """[B,T] residues. Row b takes pattern b % 7: 0 <mask> only in the last quarter; 1 <mask> only in the first quarter,
    behind left pads; 2 interior pads (also at every index in `marks` and the one before it), no <mask>; 3 every token
    a <mask>; 4 every token a pad; 5 neither; 6 trailing pads and one <mask>."""
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(4, 24, (B, T), generator=g)
    q = max(T // 4, 1)
    for b in range(B):
        k = b % 7
        if k == 0:
            tok[b, T - q::2] = mask
            if T == 1:
                tok[b, 0] = 5
        elif k == 1:
            tok[b, :q:2] = mask
            tok[b, :min(3, T - 1)] = pad
        elif k == 2:
            tok[b, 1::7] = pad
            for m in marks:
                tok[b, [i for i in (m - 1, m) if 0 <= i < T]] = pad
        elif k == 3:
            tok[b] = mask
        elif k == 4:
            tok[b] = pad
        elif k == 6:
            tok[b, T - q:] = pad
            tok[b, 0] = mask
    return tok


# ---- ESM-2 ----------------------------------------------------------------------------------------------------------
ESM2_CASES = [(1, 1, 64), (1, 3, 4), (1, 5, 320), (1, 4099, 480), (3, 1003, 2560), (7, 1003, 320), ("8sms+1", 9, 64),
              (40, 33, 5120), (14, 130, 4)]


def esm2_fp32(tok, table, token_dropout):
    """esm2.py:84-95 with the reference's fp32 tensor ops in their order; pad rows written as zeros"""
    x = table[tok]
    if token_dropout:
        x = x.masked_fill(tok.eq(MASK)[..., None], 0.0)
        ratio = tok.eq(MASK).sum(-1).float() / tok.ne(PAD).sum(-1)
        x = x * (1 - 0.15 * 0.8) / (1 - ratio)[:, None, None]
    return x.masked_fill(tok.eq(PAD)[..., None], 0.0)


@pytest.mark.parametrize("token_dropout", [1, 0], ids=["dropout", "plain"])
@pytest.mark.parametrize("B,T,E", ESM2_CASES)
def test_esm2_embed_against_float64(B, T, E, token_dropout):
    L = _lib(); lib = L.load()
    if B == "8sms+1":
        B = 8 * n_sms() + 1  # one chunk per sequence
    tok = sequence_tokens(B, T, seed=T + E).cuda()
    g = torch.Generator().manual_seed(E)
    table = torch.randn(33, E, generator=g).cuda()  # the pad row is not zero: the kernel must zero it itself
    x = torch.full((B, T, E), float("nan"), device="cuda")
    L.check(lib.esmb200_embed_tokens(P(tok), P(table), P(x), B, T, E, PAD, MASK, token_dropout, S()))
    want = kr.embed_esm2_64(tok, table, PAD, MASK, bool(token_dropout))
    pad = tok.eq(PAD)[..., None]
    if token_dropout and B > 4:
        assert bool(want[4].isnan().all())  # pads only: the reference keeps 0 / 0 ...
    want = want.masked_fill(pad, 0.0)       # ... the library writes zeros at every pad row (esmb200.h)
    assert torch.equal(x.isnan(), want.isnan())
    if B > 4:
        assert bool(x[3].isnan().all()) == bool(token_dropout) and float(x[4].abs().max()) == 0.0
    err = (x.double() - want).abs()
    bound = kr.embed_scale_bound(tok, PAD, MASK, bool(token_dropout)).cuda() * want.abs()
    if token_dropout:
        r = worst(err, bound + 1e-300)
    else:
        r = float(err.nan_to_num().max())  # exact
        assert r == 0.0
    report(f"embed_esm2 B={B} T={T} E={E} dropout={token_dropout}", err_over_bound=r)
    assert r <= 1.0
    assert same_bits(x, esm2_fp32(tok, table, token_dropout))


def test_esm2_embed_argument_checks():
    L = _lib(); lib = L.load()
    tok = torch.zeros(2, 8, dtype=torch.int64, device="cuda")
    table, x = torch.zeros(33, 8, device="cuda"), torch.zeros(2, 8, 8, device="cuda")
    before = lib.esmb200_launch_count()
    assert lib.esmb200_embed_tokens(P(tok), P(table), P(x), 2, 8, 6, PAD, MASK, 1, S()) == -1     # E % 4
    assert lib.esmb200_embed_tokens(P(tok), P(table), P(x), 0, 8, 8, PAD, MASK, 1, S()) == -1     # B = 0
    assert lib.esmb200_embed_tokens(P(tok), P(table), P(x), 65536, 8, 8, PAD, MASK, 1, S()) == -1
    assert lib.esmb200_embed_tokens(P(tok), P(table), P(x), 2, 0, 8, PAD, MASK, 1, S()) == -1     # T = 0
    assert lib.esmb200_embed_tokens(None, P(table), P(x), 2, 8, 8, PAD, MASK, 1, S()) == -1
    assert lib.esmb200_embed_tokens(P(tok), None, P(x), 2, 8, 8, PAD, MASK, 1, S()) == -1
    assert lib.esmb200_embed_tokens(P(tok), P(table), None, 2, 8, 8, PAD, MASK, 1, S()) == -1
    assert b"null argument" in lib.esmb200_last_error()
    assert lib.esmb200_launch_count() == before


# ---- ESM-1b ---------------------------------------------------------------------------------------------------------
def esm1b_rows_per_chunk(B, T):
    """the launcher's chunking (api.cu esmb200_esm1b_embed)"""
    chunks = max(min(-(-8 * n_sms() // B), -(-T // 8)), -(-T // 8192), 1)
    return -(-T // chunks)


def esm1b_run(tok, table, pos, w, b, token_dropout, pad=PAD, mask=MASK):
    L = _lib()
    B, T = tok.shape
    E = table.shape[1]
    x = torch.full((B, T, E), float("nan"), device="cuda")
    L.check(L.load().esmb200_esm1b_embed(P(tok), P(table), P(pos), P(w), P(b), 1e-5, int(token_dropout), pad, mask, P(x),
                                         B, T, E, S()))
    return x


def esm1b_check(name, tok, table, pos, w, b, token_dropout, pad=PAD, mask=MASK):
    E = table.shape[1]
    x = esm1b_run(tok, table, pos, w, b, token_dropout, pad, mask)
    want, pre = kr.embed_esm1b_64(tok, table, pos, w, b, pad, mask, bool(token_dropout))
    assert torch.equal(x.isnan(), want.isnan())  # a NaN scale (pads only, or <mask> only) spreads as in the reference
    live = tok.ne(pad) & want.isfinite().all(-1)
    assert not bool(x[tok.eq(pad) & want.isfinite().all(-1)].ne(0).any())  # finite pad rows are exact zeros
    posv = pos.double()[kr.positions(tok, pad)]
    # the sum's operands: the scaled embedding (the scale's roundings) and the position, then the sum's one rounding
    # (counted twice: a sum that rounds by exactly half an ulp sits on the bound)
    in_err = (kr.embed_scale_bound(tok, pad, mask, bool(token_dropout)).cuda() + 2 * kr.U32) * ((pre - posv).abs() + posv.abs())
    err = (x.double() - want).abs()
    if w is None:
        r = float((err[live] / (in_err[live] + 1e-300)).max())
    else:
        tol = kr.ln_tol(E, kr.row_cond(pre[live][None], tok[live][None], pad))
        r = float((err[live] / (tol * kr.ln_scale(want, w, b)[live])).max())
    report(name, err_over_bound=r, rows=float(live.sum()))
    assert r <= 1.0 and int(live.sum()) > 0
    return x


@pytest.mark.parametrize("ln", [True, False], ids=["ln", "noln"])
@pytest.mark.parametrize("token_dropout", [1, 0], ids=["dropout", "plain"])
@pytest.mark.parametrize("T,E", [(1, 128), (31, 516), (32, 1280), (33, 2560), (1026, 128), (1026, 516), (1026, 1280),
                                 (1026, 2560)])
def test_esm1b_embed_against_float64(T, E, token_dropout, ln):
    B = 7
    rows = esm1b_rows_per_chunk(B, T)
    marks = [32, 64, 96, rows, 2 * rows, 5 * rows, 37 * rows]  # ballot and chunk boundaries
    tok = sequence_tokens(B, T, seed=T + E, marks=marks).cuda()
    g = torch.Generator().manual_seed(T * E)
    table = torch.randn(33, E, generator=g).cuda()
    pos = (0.5 * torch.randn(T + PAD + 1, E, generator=g)).cuda()
    w = (1 + 0.2 * torch.randn(E, generator=g)).cuda() if ln else None
    b = (0.1 * torch.randn(E, generator=g)).cuda() if ln else None
    x = esm1b_check(f"embed_esm1b T={T} E={E} dropout={token_dropout} ln={int(ln)} rows_per_chunk={rows}", tok, table,
                    pos, w, b, token_dropout)
    if not ln and not token_dropout:  # one fp32 add, as the reference's
        ref = (table[tok] + pos[kr.positions(tok, PAD)]).masked_fill(tok.eq(PAD)[..., None], 0.0)
        assert torch.equal(x, ref)


def test_esm1b_embed_other_padding_and_mask_index():
    T, E, pad, mask = 200, 516, 3, 30
    tok = sequence_tokens(7, T, seed=5, pad=pad, mask=mask, marks=[32, 64])
    tok[0, 5::9] = tok[5, 3::4] = 1  # token 1 is a residue here
    tok = tok.cuda()
    g = torch.Generator().manual_seed(6)
    table = torch.randn(33, E, generator=g).cuda()
    pos = (0.5 * torch.randn(T + pad + 1, E, generator=g)).cuda()
    w, b = (1 + 0.2 * torch.randn(E, generator=g)).cuda(), (0.1 * torch.randn(E, generator=g)).cuda()
    esm1b_check(f"embed_esm1b T={T} E={E} padding_idx={pad} mask_idx={mask}", tok, table, pos, w, b, 1, pad, mask)


def test_esm1b_embed_longest_sequence_one_chunk_per_sequence():
    """T = 12288 (the documented limit) at B = 8 n_sms + 1, where the batch alone fills the grid: a chunk's positions
    must still fit the block's 48 KB of shared memory."""
    B, T, E = 8 * n_sms() + 1, 12288, 4
    g = torch.Generator(device="cuda").manual_seed(7)
    tok = torch.randint(4, 24, (B, T), device="cuda", generator=g)
    tok[::3, 8191:8193] = PAD
    tok[1::5, 6143:6145] = PAD
    tok[2, 12000:] = PAD
    table = torch.randn(33, E, device="cuda", generator=g)
    pos = torch.randn(T + PAD + 1, E, device="cuda", generator=g)
    x = esm1b_run(tok, table, pos, None, None, 0)
    torch.cuda.synchronize()
    ref = (table[tok] + pos[kr.positions(tok, PAD)]).masked_fill_(tok.eq(PAD)[..., None], 0.0)
    assert torch.equal(x, ref)
    report(f"embed_esm1b B={B} T={T} E={E} rows_per_chunk={esm1b_rows_per_chunk(B, T)}", max_abs_diff=0.0)


# ---- MSA Transformer ------------------------------------------------------------------------------------------------
# (E, B, R, C, msa_pos width (0: none), common offset of the tables)
MSA_CASES = [(128, 1, 1, 1, 128, 0.0), (512, 2, 3, 31, 0, 0.0), (516, 1, 3, 32, 1, 0.0), (768, 2, 3, 33, 768, 0.0),
             (1280, 1, 130, 100, 1280, 0.0), (1284, 2, 3, 100, 1284, 0.0), (2560, 2, 3, 100, 1, 0.0),
             (768, 1, 3, 1024, 768, 0.0), (128, 2, 130, 33, 1, 0.0), (2560, 1, 2, 1024, 0, 0.0),
             (768, 2, 3, 100, 768, 30.0), (4, 1, 1, 12288, 4, 0.0)]


def msa_tokens(B, R, C, seed):
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(4, 24, (B, R, C), generator=g)
    tok[:, :, 0] = 0
    if C > 3:
        tok[:, :, C - 1] = PAD        # a whole column
        tok[0, 0, 0] = PAD            # leading
    if C > 40:
        tok[:, R // 2, 30:33] = PAD   # interior, across a ballot edge
        tok[B - 1, 0, 1:40:3] = PAD
    if R > 1:
        tok[B - 1, R - 1] = PAD       # a whole row
    return tok


@pytest.mark.parametrize("E,B,R,C,width,offset", MSA_CASES)
def test_msa_embed_against_float64(E, B, R, C, width, offset):
    L = _lib(); lib = L.load()
    tok = msa_tokens(B, R, C, seed=E + C).cuda()
    g = torch.Generator().manual_seed(E * C + R)
    table = (torch.randn(33, E, generator=g) + offset).cuda()
    pos = (0.5 * torch.randn(C + PAD + 1, E, generator=g) + offset).cuda()
    mp = (0.5 * torch.randn(R + 5, width, generator=g) + offset).cuda() if width else None
    w, b = (1 + 0.2 * torch.randn(E, generator=g)).cuda(), (0.1 * torch.randn(E, generator=g)).cuda()
    x = torch.full((B, R, C, E), float("nan"), device="cuda")
    L.check(lib.esmb200_msa_embed(P(tok), P(table), P(pos), P(mp), width, P(w), P(b), 1e-5, P(x), B, R, C, E, PAD, S()))
    want, pre = kr.embed_msa_64(tok, table, pos, mp, w, b, PAD)
    assert not bool(x.isnan().any())
    live = tok.ne(PAD)
    if bool((~live).any()):
        assert float(x[~live].abs().max()) == 0.0
    cond = kr.row_cond(pre, tok, PAD)
    tol = kr.ln_tol(E, cond)
    r = float(((x.double() - want).abs()[live] / (tol * kr.ln_scale(want, w, b)[live])).max())
    report(f"embed_msa E={E} B={B} R={R} C={C} msa_pos={width} offset={offset}", err_over_bound=r, cond=cond, tol=tol)
    assert r <= 1.0
    if R > 1 and width:  # the rows of msa_pos differ, so the alignment row index matters
        assert float((mp[0] - mp[1]).abs().max()) > 1e-3


def test_msa_embed_argument_checks():
    L = _lib(); lib = L.load()
    tok = torch.zeros(1, 1, 8, dtype=torch.int64, device="cuda")
    t, x = torch.zeros(33, 8, device="cuda"), torch.zeros(1, 1, 8, 8, device="cuda")
    before = lib.esmb200_launch_count()

    def call(B=1, R=1, C=8, E=8, width=8, tokens=tok, ln=t):
        return lib.esmb200_msa_embed(P(tokens), P(t), P(t), P(t), width, P(ln), P(t), 1e-5, P(x), B, R, C, E, PAD, S())

    assert call(C=12289) == -1 and b"bad shape" in lib.esmb200_last_error()  # a row's positions would not fit
    assert call(C=0) == -1 and call(R=0) == -1 and call(B=0) == -1
    assert call(E=6) == -1 and call(E=2564) == -1
    assert call(width=4) == -1 and b"width must be E or 1" in lib.esmb200_last_error()
    assert call(tokens=None) == -1 and call(ln=None) == -1
    assert lib.esmb200_launch_count() == before
