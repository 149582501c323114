"""GPU (-m gpu): the "fp32x3" precision mode (every MMA operand an fp16 hi + lo pair, three products per MMA) and the
sharp-softmax regime VERDICT r1 asked to gate.

Why a second precision exists (scripts/precision_study.py): with q/k weights scaled
x3 the random-weight network is ill-conditioned — a 5e-4 perturbation of the residual stream grows ~10x over six layers
because near-one-hot softmaxes flip.  Emulating the roundings on the CPU shows that splitting ONLY q.k^T (the r1
verdict's proposal) moves the 6-layer error from 1.6e-2 to 1.4e-2; an exact logit path still leaves 6e-3 from the fp16
operands of the other GEMMs.  Any single-pass tensor-core evaluation (fp16, bf16 and TF32 all carry <= 11 significand
bits) is therefore outside 3e-3 in that regime; the fp32x3 mode is inside it by two orders of magnitude.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def S():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def rel_fro(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def split16(x):
    """fp32 [R,K] -> fp16 [R,2K] hi | lo (host-side statement of esmb200_convert_split)."""
    hi = x.half()
    lo = (x - hi.float()).half()
    return torch.cat((hi, lo), dim=1).contiguous()


@pytest.mark.parametrize("M,N,K", [(300, 1280, 1280), (1000, 320, 5120), (77, 3840, 640)])
def test_gemm_split_is_fp32_grade(M, N, K):
    from esm_b200 import _lib as L
    lib = L.load()
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).cuda()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).cuda()
    bias = (0.1 * torch.randn(N, generator=g)).cuda()
    ref = (a.double() @ w.double().t() + bias.double())
    a2 = torch.empty(M, 2 * K, dtype=torch.float16, device="cuda")
    w2 = torch.empty(N, 2 * K, dtype=torch.float16, device="cuda")
    L.check(lib.esmb200_convert_split(P(a), P(a2), M, K, S()))
    L.check(lib.esmb200_convert_split(P(w), P(w2), N, K, S()))
    assert torch.equal(a2, split16(a)) and torch.equal(w2, split16(w))
    out = torch.zeros(M, N, dtype=torch.float32, device="cuda")
    L.check(lib.esmb200_gemm_split(L.EPI_BIAS_F32, P(a2), P(w2), P(bias), P(out), M, N, K, None, None, 0, 0, S()))
    torch.cuda.synchronize()
    r = rel_fro(out, ref)
    fp32 = rel_fro(a @ w.t() + bias, ref)  # cuBLAS fp32 (TF32 off) on the same inputs
    print(f"PARITY gemm_split {M}x{N}x{K} rel_fro={r:.3e} (fp32 cuBLAS {fp32:.3e})")
    # the tensor cores accumulate in fp32 with truncation: the error grows like (3K/16 accumulation steps) x 2^-25, two
    # orders below the fp16 mode's 3e-4 and one above an IEEE fp32 dot product
    assert r <= 4e-5
    # fp16-output epilogue: hi | lo pair reproduces the fp32 GELU result
    if N % 64 == 0:
        out16 = torch.zeros(M, 2 * N, dtype=torch.float16, device="cuda")
        L.check(lib.esmb200_gemm_split(L.EPI_BIAS_GELU, P(a2), P(w2), P(bias), P(out16), M, N, K, None, None, 0, 0, S()))
        y = out16[:, :N].double() + out16[:, N:].double()
        want = torch.nn.functional.gelu(ref)
        assert rel_fro(y, want) <= 5e-5


def test_attention_split_is_fp32_grade():
    from esm_b200 import _lib as L
    lib = L.load()
    B, T, H = 3, 300, 4
    E = 64 * H
    g = torch.Generator().manual_seed(11)
    qkv = torch.randn(B * T, 3 * E, generator=g).cuda()
    qkv[:, :E] *= 0.125 * 4.0   # sharp logits
    qkv[:, E:2 * E] *= 4.0
    lens = torch.tensor([300, 131, 64], device="cuda")
    mask = (torch.arange(T, device="cuda")[None, :] >= lens[:, None]).to(torch.uint8).contiguous()
    q, k, v = (qkv[:, i * E:(i + 1) * E].double().view(B, T, H, 64).transpose(1, 2) for i in range(3))
    s = (q @ k.transpose(-1, -2)).masked_fill(mask.bool()[:, None, None, :], float("-inf"))
    p = torch.softmax(s, -1)
    ref = (p @ v).transpose(1, 2).reshape(B * T, E)
    qkv2 = split16(qkv)                       # [q k v]_hi | [q k v]_lo
    ctx = torch.zeros(B * T, 2 * E, dtype=torch.float16, device="cuda")
    probs = torch.zeros(B, H, T, T, dtype=torch.float32, device="cuda")
    scratch = torch.empty(lib.esmb200_attention_scratch_bytes(B, T), dtype=torch.uint8, device="cuda")
    L.check(lib.esmb200_attention_split(P(qkv2), P(mask), P(ctx), P(probs), B, T, H, P(scratch), S()))
    torch.cuda.synchronize()
    valid = (torch.arange(T, device="cuda")[None, :] < lens[:, None]).reshape(-1)
    got = ctx[:, :E].double() + ctx[:, E:].double()
    r = rel_fro(got[valid], ref[valid])
    pa = float((probs.double() - p)[valid.view(B, T)[:, None, :, None].expand_as(p)].abs().max())
    print(f"PARITY attention_split rel_fro={r:.3e} probs_max_abs={pa:.3e}")
    assert r <= 1e-5 and pa <= 3e-5


def _models(L_, E, H, gain):
    from esm_b200 import ESM2
    from oracle.weights import make_state_dict
    sd = make_state_dict(L_, E, H, seed=0, qk_gain=gain)
    model = ESM2(num_layers=L_, embed_dim=E, attention_heads=H)
    model.load_state_dict(sd, strict=True)
    return model.eval().cuda(), sd


@pytest.mark.parametrize("gain", [1.5, 3.0])
def test_sharp_softmax_regime_six_layers_650M_width(gain):
    """VERDICT r1 next-round item 1(b): qk_gain = 3.0 (softmax close to one-hot), 6 layers at the 650M width, gated at
    rel-Frobenius <= 3e-3 and attention max-abs <= 1e-2 — met by the fp32x3 mode; the fp16 mode is held to its measured
    conditioning-limited bound (and to the normal tolerance at the default gain)."""
    from oracle import esm2_oracle
    from oracle.weights import make_tokens
    L_, E, H = 6, 1280, 20
    model, sd = _models(L_, E, H, gain)
    tokens = make_tokens([254, 180], 256, seed=5)
    ref = esm2_oracle.esm2_forward(sd, L_, H, tokens, repr_layers=[L_], need_head_weights=True)
    res = {}
    for prec in ("fp16", "fp32x3"):
        model.set_precision(prec)
        out = model(tokens.cuda(), repr_layers=[L_], need_head_weights=True)
        torch.cuda.synchronize()
        r = rel_fro(out["representations"][L_].cpu(), ref["representations"][L_])
        a = float((out["attentions"].cpu() - ref["attentions"]).abs().max())
        lg = rel_fro(out["logits"].cpu(), ref["logits"])
        res[prec] = (r, a, lg)
        print(f"PARITY sharp gain={gain} {prec}: repr rel_fro={r:.3e} attn max_abs={a:.3e} logits rel_fro={lg:.3e}")
    r, a, lg = res["fp32x3"]
    assert r <= 3e-3 and a <= 1e-2 and lg <= 4e-3          # the gate
    assert r <= 1e-3 and a <= 5e-3                         # measured 1.8e-4 / 2.1e-3 at gain 3, 1.9e-5 / 5e-5 at gain 1.5
    r16, a16, _ = res["fp16"]
    if gain <= 1.5:
        assert r16 <= 3e-3 and a16 <= 1e-2                 # the stated fp16 tolerance (DESIGN.md section 4)
    else:
        assert r16 <= 4e-2                                 # ill-conditioned regime: measured 1.4e-2, see the docstring


def test_fp32x3_small_models_and_contacts_vs_reference_golden(golden_dir):
    """the whole model in fp32x3 against the committed reference outputs: error two orders below the fp16 mode."""
    import os
    for name in ("mid_L3_E256_H4", "t6_8M_like_L6_E320_H20"):
        fx = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
        cfg = fx["config"]
        model, _ = _models(cfg["num_layers"], cfg["embed_dim"], cfg["attention_heads"], 1.5)
        model.set_precision("fp32x3")
        out = model(fx["tokens"].cuda(), repr_layers=fx["repr_layers"], return_contacts=True)
        torch.cuda.synchronize()
        k = cfg["num_layers"]
        r = rel_fro(out["representations"][k].cpu(), fx["representations"][k])
        lg = rel_fro(out["logits"].cpu(), fx["logits"])
        c = float((out["contacts"].cpu() - fx["contacts"]).abs().max())
        print(f"PARITY fp32x3 {name}: repr rel_fro={r:.3e} logits={lg:.3e} contacts max_abs={c:.3e}")
        assert r <= 2e-5 and lg <= 2e-5 and c <= 1e-4
