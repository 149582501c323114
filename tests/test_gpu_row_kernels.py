"""GPU (-m gpu): the LayerNorm row kernel (layernorm_rows_kernel, fp32 / fp16 / fp32x3-split outputs) against float64
at the widths where its register tiling has edges, in place, and on rows with a large mean; and programmatic dependent
launch (esmb200_set_option("pdl", 1)), which must not change any output."""
import pytest
import torch

import fp8_refs as fr
import kernel_refs as kr

pytestmark = pytest.mark.gpu


def _lib():
    from esm_b200 import _lib
    return _lib


def S():
    return torch.cuda.current_stream().cuda_stream


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def ln_inputs(M, E, seed, mean=0.5, std=3.0):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(M, E, generator=g, dtype=torch.float64) * std + mean).float().cuda()
    w = (1 + 0.2 * torch.randn(E, generator=g)).cuda()
    b = (0.1 * torch.randn(E, generator=g)).cuda()
    return x, w, b


# fp32 output, relative to |g| (|xhat| + 1) + |b| (xhat the normalised row): the two-pass mean and variance of E fp32
# values (a rounding walk of ~sqrt(E) steps of u |partial sum|, so |d mean| / std <~ sqrt(E) u |mean| / std), rsqrt
# (2 ulp) and the affine step (3 roundings): 4 u (8 + 2 sqrt(E) (1 + |mean| / std)) with a factor 4 of room. fp16
# outputs add half an fp16 ulp (2^-11); the split output hi + lo carries 22 bits. At mean 1e3, std 0.1 the bound is
# loose (measured 1e-3 .. 2e-3 against 1e-2 .. 0.34): there it stands guard against a one-pass E[x^2] - mean^2
# variance, which loses the whole variance in fp32 at that ratio.
#
# The e4m3 output (esmb200_layernorm_fp8, OUT = 3) is checked against fr.quantize of the float64 LayerNorm, with the
# same bound per element (tol_f32 times the scale above): a scale may differ by one power of two only where the block's
# float64 amax lies within that bound of an edge 448 2^k, a code under an equal scale only where y / s lies within it
# of a rounding midpoint (fp8_refs.check_codes).  E = 132 and 260 end in a 4-column block (one lane's float4); the
# scales are read in their [ceil(E/128), M] layout from inside guard bands; M = 37 is not a multiple of the 8 rows
# (warps) of a CTA.  A second call with gamma = beta = 0 over one 128-column block must give that block scale 1 and
# code 0, and every other block the first call's bits (gamma and beta do not enter the row statistics).
@pytest.mark.parametrize("E", [4, 96, 132, 260, 480, 512, 516, 1280, 1284, 2560, 2564, 5120])
@pytest.mark.parametrize("big_mean", [False, True], ids=["mean0.5_std3", "mean1e3_std0.1"])
def test_layernorm_widths_against_float64(E, big_mean):
    L = _lib(); lib = L.load()
    M = 37
    x, w, b = ln_inputs(M, E, seed=E, **({"mean": 1e3, "std": 0.1} if big_mean else {}))
    want = kr.layer_norm64(x, w, b)
    cond = 1e4 if big_mean else 1.0  # |mean| / std
    tol = 4 * kr.U32 * (8 + 2 * E ** 0.5 * (1 + cond))
    scale = (want - b.double()).abs() + w.double().abs() + b.double().abs()
    q8, qbuf = fr.guarded((M, E), torch.uint8, "cuda")
    s8, sbuf = fr.guarded((-(-E // 128), M), torch.float32, "cuda")
    L.check(lib.esmb200_layernorm_fp8(x.data_ptr(), w.data_ptr(), b.data_ptr(), q8.data_ptr(), s8.data_ptr(), M, E,
                                      1e-5, S()))
    torch.cuda.synchronize()
    assert fr.guard_changes(qbuf) == 0 and fr.guard_changes(sbuf) == 0
    assert not bool(((q8 & 0x7F) == 0x7F).any()) and not bool(s8.isnan().any())
    r8 = fr.check_codes(q8.cpu().view(torch.float8_e4m3fn), s8, want, tol * scale)
    report(f"layernorm_fp8 E={E} {'mean1e3_std0.1' if big_mean else 'mean0.5_std3'}", flips=r8["flips"],
           scale_flips=r8["scale_flips"], n=r8["n"])
    assert r8["bad_scale"] == 0 and r8["bad_code"] == 0, r8
    # a flip needs y / s within the bound of a midpoint.  Measured on an H100: no flip at mean 0.5 / std 3; at mean 1e3
    # / std 0.1, where the bound reaches 0.34 of the scale above and the window alone would admit almost any code, up
    # to 2.7 % of the elements (the fp32 mean's rounding walk), against a ceiling of 5 %
    assert r8["flips"] <= (max(64, r8["n"] // 50) if not big_mean else r8["n"] // 20), r8
    if E >= 256:
        zb = 1  # the second 128-column block
        w0, b0 = w.clone(), b.clone()
        w0[128 * zb:128 * zb + 128] = 0
        b0[128 * zb:128 * zb + 128] = 0
        q0 = torch.full_like(q8, 0xFF)
        s0 = torch.full_like(s8, float("nan"))
        L.check(lib.esmb200_layernorm_fp8(x.data_ptr(), w0.data_ptr(), b0.data_ptr(), q0.data_ptr(), s0.data_ptr(), M,
                                          E, 1e-5, S()))
        torch.cuda.synchronize()
        blk = slice(128 * zb, 128 * zb + 128)
        assert bool((s0[zb] == 1.0).all()) and bool((q0[:, blk] == 0).all())
        rest = torch.ones(E, dtype=torch.bool, device="cuda")
        rest[blk] = False
        assert torch.equal(q0[:, rest], q8[:, rest])
        assert torch.equal(torch.cat([s0[:zb], s0[zb + 1:]]), torch.cat([s8[:zb], s8[zb + 1:]]))
    out = torch.full_like(x, float("nan"))
    L.check(lib.esmb200_layernorm(x.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), M, E, 1e-5, S()))
    out16 = torch.full((M, E), float("nan"), dtype=torch.float16, device="cuda")
    L.check(lib.esmb200_layernorm_f16(x.data_ptr(), w.data_ptr(), b.data_ptr(), out16.data_ptr(), M, E, 1e-5, S()))
    split = torch.full((M, 2 * E), float("nan"), dtype=torch.float16, device="cuda")
    L.check(lib.esmb200_layernorm_split(x.data_ptr(), w.data_ptr(), b.data_ptr(), split.data_ptr(), M, E, 1e-5, S()))
    e32 = float(((out.double() - want).abs() / scale).max())
    e16 = float(((out16.double() - want).abs() / scale).max())
    esp = float(((split[:, :E].double() + split[:, E:].double() - want).abs() / scale).max())
    report(f"layernorm E={E} {'mean1e3_std0.1' if big_mean else 'mean0.5_std3'}", f32_rel=e32, f16_rel=e16,
           split_rel=esp, tol_f32=tol)
    assert e32 <= tol and esp <= tol + 2.0 ** -22
    assert e16 <= tol + 2.0 ** -11
    assert torch.equal(out16, out.half())  # the fp16 output is the fp32 result rounded to nearest


@pytest.mark.parametrize("E", [96, 1280, 5120])
def test_layernorm_in_place(E):
    """out aliasing x (the final LayerNorm of the model runs so): the same bits as out-of-place."""
    L = _lib(); lib = L.load()
    M = 300
    x, w, b = ln_inputs(M, E, seed=E + 1)
    ref = torch.empty_like(x)
    L.check(lib.esmb200_layernorm(x.data_ptr(), w.data_ptr(), b.data_ptr(), ref.data_ptr(), M, E, 1e-5, S()))
    L.check(lib.esmb200_layernorm(x.data_ptr(), w.data_ptr(), b.data_ptr(), x.data_ptr(), M, E, 1e-5, S()))
    assert torch.equal(x, ref)


def _msa_inputs():
    """Two axial layers at E = 128 and a [B,R,C,E] input with padded columns in the second alignment."""
    from argparse import Namespace
    from esm_b200.msa import MSATransformer
    from oracle.msa_oracle import make_msa_state_dict
    E, F, H = 128, 256, 2
    m = MSATransformer(Namespace(layers=2, embed_dim=E, ffn_embed_dim=F, attention_heads=H, max_positions=1024,
                                 embed_positions_msa=True))
    m.load_state_dict(make_msa_state_dict(2, E, F, H, seed=3), strict=True)
    m = m.eval().cuda()
    B, R, C = 2, 5, 70
    x = torch.randn(B, R, C, E, generator=torch.Generator().manual_seed(3)).cuda()
    pad = torch.zeros(B, R, C, dtype=torch.bool)
    pad[1, :, C - 9:] = True
    return list(m.layers), x, pad.cuda()


def test_pdl_changes_no_output():
    """One ESM-2 forward with representations, attentions and contacts, and one MSA axial stack forward
    (esmb200_axial_stack_forward), with programmatic dependent launch on and off: identical results."""
    from esm_b200 import ESM2
    from esm_b200.msa import run_axial_stack
    from oracle.weights import make_state_dict, make_tokens
    L = _lib(); lib = L.load()
    model = ESM2(num_layers=3, embed_dim=256, attention_heads=4)
    model.load_state_dict(make_state_dict(3, 256, 4, seed=2), strict=True)
    model = model.eval().cuda()
    tokens = make_tokens([150, 77, 9], 152, seed=2, n_mask=2).cuda()
    layers, x0, pad = _msa_inputs()

    def run_all():
        with torch.no_grad():
            out = model(tokens, repr_layers=[0, 1, 3], return_contacts=True)
            x = x0.clone()
            row = run_axial_stack(layers, x, pad, row_attn_layers=[0, 1])
        torch.cuda.synchronize()
        reps = [out["representations"][k] for k in (0, 1, 3)]
        return [out["logits"], out["attentions"], out["contacts"]] + reps + [x, row[0], row[1]]

    try:
        L.check(lib.esmb200_set_option(b"pdl", 0))
        off = run_all()
        L.check(lib.esmb200_set_option(b"pdl", 1))
        on = run_all()
    finally:
        L.check(lib.esmb200_set_option(b"pdl", 0))
    for i, (a, b) in enumerate(zip(off, on)):
        assert torch.equal(a, b), i
