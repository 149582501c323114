"""GPU (-m gpu): the fp16 tied row attention of the MSA Transformer (esmb200_tied_row_attention: tied_scores_kernel,
tied_softmax_kernel, tied_pv_kernel <false>) against float64 torch on the fp16-rounded q, k, v, at the shapes where the
kernels have edges: C not a multiple of 64 / 128 (boxes that read into the next alignment row, zero P columns in
[C, Cp)), R not a multiple of the four alignment rows a P.V CTA handles, C = 1, C = 1024 (the softmax's register
limit), R = 1024 (the longest K chain of the logits), key padding, an alignment whose key columns are all padded, and
the call without probabilities (the logits then live in scratch)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _lib():
    from esm_b200 import _lib
    return _lib


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def inputs(B, R, C, H, seed, pad_cols=0, pad_all=None):
    """fp16 qkv [B*R*C, 3E] with q scaled so that the summed logits have std ~3, and key_pad [B,C] (uint8) or None.
    q is zeroed at padded columns, as the MSA layer does (axial_attention.py:82-85)."""
    g = torch.Generator().manual_seed(seed)
    E = 64 * H
    q = torch.randn(B, R, C, H, 64, generator=g) * (3.0 / (R * 64) ** 0.5)
    k = torch.randn(B, R, C, H, 64, generator=g)
    v = torch.randn(B, R, C, H, 64, generator=g)
    pad = None
    if pad_cols or pad_all is not None:
        pad = torch.zeros(B, C, dtype=torch.bool)
        if pad_cols:
            pad[:, C - pad_cols:] = True
            pad[0, C // 3] = True
        if pad_all is not None:
            pad[pad_all] = True
        q = q * (~pad)[:, None, :, None, None]
    qkv = torch.cat([t.reshape(B * R * C, E) for t in (q, k, v)], 1).half().cuda()
    return qkv, (pad.to(torch.uint8).cuda() if pad is not None else None)


def reference(qkv, pad, B, R, C, H):
    """float64 on the fp16 operands: logits summed over the rows, -10000 at padded keys, softmax, P.V."""
    y = qkv.double().view(B, R, C, 3, H, 64)
    q, k, v = y[:, :, :, 0], y[:, :, :, 1], y[:, :, :, 2]
    logits = torch.einsum("brihd,brjhd->hbij", q, k)
    if pad is not None:
        logits = logits.masked_fill(pad.bool()[None, :, None, :], -10000)
    p = logits.softmax(-1)
    return torch.einsum("hbij,brjhd->brihd", p, v).reshape(B * R * C, H * 64), p


def run(qkv, pad, B, R, C, H, probs=True):
    L = _lib(); lib = L.load()
    E = 64 * H
    nbytes = lib.esmb200_tied_row_attention_scratch_bytes(B, C, H)
    scratch = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")  # NaN-filled logits / P
    ctx = torch.full((B * R * C, E), float("nan"), dtype=torch.float16, device="cuda")
    p = torch.full((H, B, C, C), float("nan"), device="cuda") if probs else None
    rc = lib.esmb200_tied_row_attention(qkv.data_ptr(), pad.data_ptr() if pad is not None else None, ctx.data_ptr(),
                                        p.data_ptr() if probs else None, B, R, C, H, scratch.data_ptr(), nbytes,
                                        torch.cuda.current_stream().cuda_stream)
    L.check(rc)
    return ctx, p


# Tolerances. Probabilities: the logits are fp32 sums of R*64 fp16 products (exact products, truncating tensor-core
# accumulation: |ds| <~ (R*64/16) 2^-23 |s|max at worst, ~1e-5 at std 3 and R <= 7, ~3e-4 at R = 1024); |dp| <= 2 p |ds|
# plus __expf's 2 ulp: atol 2e-5 + rtol 2e-4 as for the flash kernels, rtol 1e-3 at R = 1024.
# Context: P is rounded to fp16 before P.V, |dctx| <= 2^-11 max|v| sum_j p_j ~ 2.4e-3 for |v| <= 5, plus half an fp16
# ulp of the output (2.4e-4 at |ctx| <= 1): atol 4e-3.
SHAPES = [(1, 1, 1, 1), (2, 3, 64, 2), (1, 5, 65, 1), (1, 7, 127, 2), (2, 6, 128, 4), (1, 2, 129, 12),
          (1, 2, 1024, 1), (1, 1024, 64, 2)]


@pytest.mark.parametrize("B,R,C,H", SHAPES)
def test_tied_row_attention_against_float64(B, R, C, H):
    qkv, _ = inputs(B, R, C, H, seed=B * 7919 + R * 31 + C)
    ctx, p = run(qkv, None, B, R, C, H)
    want, pwant = reference(qkv, None, B, R, C, H)
    ce, pe = float((ctx.double() - want).abs().max()), float((p.double() - pwant).abs().max())
    report(f"tied_row fp16 (B,R,C,H)=({B},{R},{C},{H})", ctx_max_abs=ce, probs_max_abs=pe)
    torch.testing.assert_close(p.double(), pwant, atol=2e-5, rtol=1e-3 if R >= 1024 else 2e-4)
    torch.testing.assert_close(ctx.double(), want, atol=4e-3, rtol=0)
    # without probabilities (logits in scratch) the context is the same bits
    ctx2, _ = run(qkv, None, B, R, C, H, probs=False)
    assert torch.equal(ctx, ctx2)


@pytest.mark.parametrize("pad_cols", [0, 40])
def test_tied_row_attention_with_key_padding(pad_cols):
    B, R, C, H = 3, 6, 300, 2
    qkv, pad = inputs(B, R, C, H, seed=11 + pad_cols, pad_cols=pad_cols)
    if pad is None:
        pad = torch.zeros(B, C, dtype=torch.uint8, device="cuda")  # a key_pad with nothing padded
    ctx, p = run(qkv, pad, B, R, C, H)
    want, pwant = reference(qkv, pad, B, R, C, H)
    ce, pe = float((ctx.double() - want).abs().max()), float((p.double() - pwant).abs().max())
    report(f"tied_row fp16 key_pad (B,R,C,H)=({B},{R},{C},{H}) pad_cols={pad_cols}", ctx_max_abs=ce, probs_max_abs=pe)
    torch.testing.assert_close(p.double(), pwant, atol=2e-5, rtol=2e-4)
    torch.testing.assert_close(ctx.double(), want, atol=4e-3, rtol=0)
    ctx2, _ = run(qkv, pad, B, R, C, H, probs=False)
    assert torch.equal(ctx, ctx2)


def test_tied_row_attention_all_keys_padded():
    """Every key column of alignment 1 is padded: all its logits are -10000 and the softmax is uniform, 1 / C."""
    B, R, C, H = 2, 3, 130, 2
    qkv, pad = inputs(B, R, C, H, seed=5, pad_all=1)
    ctx, p = run(qkv, pad, B, R, C, H)
    want, pwant = reference(qkv, pad, B, R, C, H)
    assert float((pwant[:, 1] - 1.0 / C).abs().max()) < 1e-15
    report("tied_row fp16 all keys padded", ctx_max_abs=float((ctx.double() - want).abs().max()),
           probs_max_abs=float((p.double() - pwant).abs().max()))
    torch.testing.assert_close(p.double(), pwant, atol=2e-5, rtol=2e-4)
    torch.testing.assert_close(ctx.double(), want, atol=4e-3, rtol=0)


def test_tied_row_attention_rejects_more_than_1024_columns():
    L = _lib(); lib = L.load()
    B, R, C, H = 1, 1, 1025, 1
    qkv = torch.zeros(B * R * C, 3 * 64 * H, dtype=torch.float16, device="cuda")
    ctx = torch.empty(B * R * C, 64 * H, dtype=torch.float16, device="cuda")
    nbytes = lib.esmb200_tied_row_attention_scratch_bytes(B, C, H)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    rc = lib.esmb200_tied_row_attention(qkv.data_ptr(), None, ctx.data_ptr(), None, B, R, C, H, scratch.data_ptr(),
                                        nbytes, torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and b"1024" in lib.esmb200_last_error()
