"""GPU (-m gpu): the "fp8" precision — e4m3 block-scaled QKV, fc1 and fc2 GEMMs (gemm_fp8.cuh).

Kernel level: the quantisers equal torch.float8_e4m3fn bit for bit; the GEMM equals the float64 product of the
dequantised operands within the accumulation bound below, for every model's (N, K) and every epilogue.  Layer and model
level: every layer of an fp8 forward matches a float64 emulation of the same quantisation steps (fp8_refs.emulate_layer),
every committed golden also stays close to the reference, fused contacts equal the contact head on the same run's
attentions, the variant scorers equal the forward on the masked copies, and switching back to fp16 reproduces fp16 bit
for bit.
"""
import ctypes
import glob
import math
import os

import pytest
import torch

import fp8_refs as fr

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def P(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def S():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def lib():
    from esm_b200 import _lib
    return _lib, _lib.load()


def quantize_dev(x, block_rows):
    L, lb = lib()
    R, K = x.shape
    q = torch.empty(R, K, dtype=torch.uint8, device="cuda")
    s = torch.empty(*((-(-K // 128), R) if block_rows == 1 else (-(-R // 128), -(-K // 128))), device="cuda")
    L.check(lb.esmb200_quantize_fp8(P(x), P(q), P(s), R, K, block_rows, S()))
    return q, s


@pytest.mark.parametrize("block_rows", [1, 128])
@pytest.mark.parametrize("R,K", [(1, 320), (129, 480), (300, 1280), (257, 5120)])
def test_quantizers_bit_exact(block_rows, R, K):
    g = torch.Generator().manual_seed(R * K + block_rows)
    x = torch.randn(R, K, generator=g) * torch.exp(4 * torch.randn(R, 1, generator=g))
    x[0, :128] = 0.0                       # an all-zero block (scale 1) in the first K block
    x[-1, -5:] = 448.0 * 2.0 ** -3         # an exact power-of-two amax boundary
    x[R // 2, 1] = -1e-30                  # far below the block's amax: an e4m3 subnormal / zero
    q, s = quantize_dev(x.cuda(), block_rows)
    qr, sr = fr.quantize(x, block_rows)
    assert torch.equal(s.cpu(), sr)
    assert torch.equal(q.cpu(), qr.view(torch.uint8))


def test_layernorm_fp8():
    L, lb = lib()
    for M, E in [(5, 320), (130, 480), (64, 1280), (8, 5120)]:
        g = torch.Generator().manual_seed(M + E)
        x = (torch.randn(M, E, generator=g) * 3).cuda()
        w, b = (1 + 0.1 * torch.randn(E, generator=g)).cuda(), (0.1 * torch.randn(E, generator=g)).cuda()
        q = torch.empty(M, E, dtype=torch.uint8, device="cuda")
        s = torch.empty(-(-E // 128), M, device="cuda")
        L.check(lb.esmb200_layernorm_fp8(P(x), P(w), P(b), P(q), P(s), M, E, 1e-5, S()))
        y = torch.nn.functional.layer_norm(x.double(), (E,), w.double(), b.double(), 1e-5).cpu()
        deq = fr.dequantize(q.cpu().view(torch.float8_e4m3fn), s.cpu(), 1)
        sfull = s.cpu().t().double().repeat_interleave(128, 1)[:, :E]
        # e4m3 keeps 3 significand bits: half an ulp is 2^-4 relative, 2^-10 * s below the normal range (2^-6 s)
        bound = torch.maximum(y.abs() * 2.0 ** -4, sfull * 2.0 ** -10) * (1 + 1e-3) + 1e-6 * y.abs()
        assert bool(((deq - y).abs() <= bound).all())


# every model's (N, K) of the three fp8 projections: QKV [3 Ea, E], fc1 [4E, E], fc2 [E, 4E]; 8M and 35M have partial
# 128-wide K blocks (E = 320, 480), 15B is the largest
MODELS = {"8M": (320, 1280), "35M": (480, 1280), "150M": (640, 1280), "650M": (1280, 1280), "3B": (2560, 2560),
          "15B": (5120, 5120)}


def shapes(model):
    E, Ea = MODELS[model]
    return {"qkv": (3 * Ea, E), "fc1": (4 * E, E), "fc2": (E, 4 * E)}


def operands(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) * K ** -0.5
    bias = 0.1 * torch.randn(N, generator=g)
    qa, sa = quantize_dev(a.cuda(), 1)
    qw, sw = quantize_dev(w.cuda(), 128)
    A = fr.dequantize(qa.cpu().view(torch.float8_e4m3fn), sa.cpu(), 1).cuda()
    W = fr.dequantize(qw.cpu().view(torch.float8_e4m3fn), sw.cpu(), 128).cuda()
    return qa, sa, qw, sw, bias.cuda(), A, W


def acc_bound(A, W):
    """|kernel accumulator - A.W^T| per element.  Each 128-wide K block is 4 wgmma k32 steps on the fp8 tensor cores,
    whose internal sum keeps at least 13 significand bits (DeepSeek-V3 section 3.3.2 measured about 14): the block's
    error is at most 2^-12 of its sum of |products|; the promotion into the fp32 accumulator adds 2^-24 of the running
    sum per block.  Both are bounded by 2^-12 (1 + 2^-12 K/128) |A|.|W|^T."""
    K = A.shape[1]
    return (A.abs() @ W.abs().t()) * (2.0 ** -12 * (1 + 2.0 ** -12 * math.ceil(K / 128))) + 1e-30


def gelu64(x):
    return x * 0.5 * (1 + torch.erf(x / math.sqrt(2)))


M_ALL = [1, 127, 128, 129, 4097]
CASES = ([("650M", "fc1", M) for M in M_ALL] + [("650M", "fc2", M) for M in M_ALL] + [("650M", "qkv", M) for M in M_ALL]
         + [(m, p, 129) for m in MODELS for p in ("qkv", "fc1", "fc2")]
         + [(m, p, 4097) for m in ("8M", "35M", "15B") for p in ("qkv", "fc1", "fc2")])


@pytest.mark.parametrize("model,proj,M", CASES)
def test_gemm_fp8(model, proj, M):
    L, lb = lib()
    N, K = shapes(model)[proj]
    qa, sa, qw, sw, bias, A, W = operands(M, N, K, seed=M * 7 + N + K)
    ref = A @ W.t() + bias.double()
    bnd = acc_bound(A, W)
    if proj == "fc2":  # EPI_BIAS_RESIDUAL: out += y
        x0 = torch.randn(M, N, device="cuda")
        out = x0.clone()
        L.check(lb.esmb200_gemm_fp8(L.EPI_BIAS_RESIDUAL, P(qa), P(sa), P(qw), P(sw), P(bias), P(out), None, M, N, K,
                                    None, None, 0, 0, S()))
        torch.cuda.synchronize()
        y = out.double() - x0.double()
        # two fp32 roundings (y, then x + y) on top of the accumulation bound
        tol = bnd + 2.0 ** -23 * (ref.abs() + x0.double().abs()) * 2
        ratio = float(((y - ref).abs() / tol).max())
    elif proj == "qkv":  # EPI_QKV_ROPE -> fp16, rope tables over T = 64 positions
        E = N // 3
        T = 64
        inv = 1.0 / (10000 ** (torch.arange(0, 64, 2).double() / 64))
        ang = torch.arange(T).double()[:, None] * inv[None]
        cos, sin = ang.cos().float().cuda(), ang.sin().float().cuda()
        out = torch.empty(M, N, dtype=torch.float16, device="cuda")
        L.check(lb.esmb200_gemm_fp8(L.EPI_QKV_ROPE, P(qa), P(sa), P(qw), P(sw), P(bias), P(out), None, M, N, K,
                                    P(cos), P(sin), T, E, S()))
        torch.cuda.synchronize()
        y = ref.clone()
        y[:, :E] *= 0.125
        t = torch.arange(M, device="cuda") % T
        c, s = cos.double()[t], sin.double()[t]
        for sect in (0, 1):  # rotate-half inside every 64-wide slot: column j pairs with j + 32
            v = y[:, sect * E:(sect + 1) * E].view(M, -1, 2, 32)
            a0, b0 = v[:, :, 0].clone(), v[:, :, 1].clone()
            v[:, :, 0] = a0 * c[:, None] - b0 * s[:, None]
            v[:, :, 1] = b0 * c[:, None] + a0 * s[:, None]
        b2 = bnd.clone()
        b2[:, :E] *= 0.125
        b2[:, :2 * E] *= 2  # a rotated value mixes two accumulators
        tol = b2 + 2.0 ** -11 * y.abs() + 2.0 ** -24
        ratio = float(((out.double() - y).abs() / tol).max())
    else:  # fc1: EPI_GELU_FP8 -> e4m3 + one scale per row and 128 columns
        out = torch.empty(M, N, dtype=torch.uint8, device="cuda")
        so = torch.empty(N // 128, M, device="cuda")
        L.check(lb.esmb200_gemm_fp8(L.EPI_GELU_FP8, P(qa), P(sa), P(qw), P(sw), P(bias), P(out), P(so), M, N, K,
                                    None, None, 0, 0, S()))
        torch.cuda.synchronize()
        y = gelu64(ref)
        qr, sr = fr.quantize(y.float().cpu(), 1)
        q8 = out.cpu().view(torch.float8_e4m3fn)
        # the scale flips only where the block's amax lies within the accumulation bound of a scale boundary
        # |GELU'| <= 1.13; the kernel's erf (Abramowitz & Stegun 7.1.26) is within 1.5e-7 absolute, i.e. x/2 * 1.5e-7
        # on GELU(x); its ex2 / rcp approximations and the fp32 bias add stay within 2^-20 relative
        ybnd = (bnd * 1.13 + 1e-7 * ref.abs() + 2.0 ** -20 * y.abs()).cpu()
        sflip = so.cpu() != sr
        deq = fr.dequantize(q8, so.cpu(), 1)
        mism = (q8.view(torch.uint8) != qr.view(torch.uint8)) | sflip.t().repeat_interleave(128, 1)[:, :N]
        # a code mismatch under the same scale must be a rounding-boundary flip: the kernel's code is the e4m3 rounding
        # of a value within the bound of the float64 one (half an e4m3 ulp: 2^-4 relative, 2^-10 s for subnormals)
        same_s = ~sflip.t().repeat_interleave(128, 1)[:, :N]
        sfull = so.cpu().t().double().repeat_interleave(128, 1)[:, :N]
        half_ulp = torch.maximum(deq.abs() * 2.0 ** -4, sfull * 2.0 ** -10)
        flip_ok = (y.cpu() - deq).abs() <= half_ulp * (1 + 1e-6) + ybnd
        bad = mism & ~flip_ok  # every code, also in blocks whose scale differs, within the bound after dequantising
        nflip = int((mism & same_s).sum())
        print(f"FP8 gemm gelu {model} {proj} M={M}: {nflip} boundary flips of {M * N}, {int(sflip.sum())} scale flips")
        assert int(bad.sum()) == 0
        assert nflip <= max(64, M * N // 50)  # measured on an H100: 0.5-0.7 % of the elements
        ratio = 0.0
        if bool(sflip.any()):
            # a scale differs by one power of two, and only where the block's float64 amax lies within the bound of
            # the boundary 448 * min(s, s') between the two scales (plus the fp32 rounding of the amax)
            assert bool((sr[sflip] / so.cpu()[sflip]).log2().abs().eq(1).all())
            am = y.abs().cpu().view(M, N // 128, 128).amax(-1).t()
            bmax = ybnd.view(M, N // 128, 128).amax(-1).t()
            edge = 448 * torch.minimum(sr, so.cpu()).double()
            assert bool(((am - edge).abs()[sflip] <= bmax[sflip] + 2.0 ** -23 * am[sflip]).all())
    print(f"FP8 gemm {model} {proj} M={M} N={N} K={K}: max err / bound = {ratio:.3f}")
    assert ratio <= 1.0


def build(L, E, H, seed=0):
    from esm_b200 import ESM2
    from oracle.weights import make_state_dict
    m = ESM2(num_layers=L, embed_dim=E, attention_heads=H)
    m.load_state_dict(make_state_dict(L, E, H, seed=seed), strict=True)
    return m.eval().cuda()


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


GOLDENS = sorted(p for p in glob.glob(os.path.join(GOLDEN, "*.pt")) if not os.path.basename(p).startswith("msa"))


@pytest.mark.parametrize("path", GOLDENS, ids=os.path.basename)
def test_goldens_in_fp8(path):
    g = torch.load(path, weights_only=False)
    cfg = g["config"]
    r0, r1 = g.get("rows", (0, g["tokens"].shape[1]))
    if os.path.basename(path).startswith("esm1b"):
        import argparse
        from esm_b200 import ProteinBertModel
        from esm1b_weights import make_esm1b_state_dict
        args = argparse.Namespace(**cfg["model_args"])
        model = ProteinBertModel(args, "roberta_large")
        model.load_state_dict(make_esm1b_state_dict(cfg["num_layers"], cfg["embed_dim"], cfg["attention_heads"],
                                                    seed=cfg["seed"], emb_layer_norm_before=args.emb_layer_norm_before))
        model = model.eval().cuda()
    else:
        model = build(cfg["num_layers"], cfg["embed_dim"], cfg["attention_heads"], cfg.get("seed", 0))
    tok = g["tokens"].cuda()
    out16 = model(tok, repr_layers=g["repr_layers"])
    model.set_precision("fp8")
    out8 = model(tok, repr_layers=g["repr_layers"])
    check_against_emulation(model, tok, os.path.basename(path))  # tight: the same quantisation steps in float64
    model.set_precision("fp16")
    back = model(tok, repr_layers=g["repr_layers"])
    assert torch.equal(back["logits"], out16["logits"])  # switching back re-packs the same fp16 operands
    for k in g["repr_layers"]:
        assert torch.equal(back["representations"][k], out16["representations"][k])
    e8 = rel(out8["logits"][:, r0:r1].cpu(), g["logits"])
    e16 = rel(out16["logits"][:, r0:r1].cpu(), g["logits"])
    last = max(g["repr_layers"])
    r8 = rel(out8["representations"][last][:, r0:r1].cpu(), g["representations"][last])
    print(f"FP8 golden {os.path.basename(path)}: logits rel {e8:.3e} (fp16 {e16:.3e}), repr[{last}] rel {r8:.3e}")
    # loose, against the fp32 reference (the tight check is the emulation above): e4m3 carries 3 significand bits, each
    # quantised operand is within 2^-4 relative (about 3.6 % RMS), and three of the layer's five GEMMs quantise two
    # operands; measured on an H100: 4.3-12.0 % on the logits, 4.3-9.8 % on the last representation (6-layer 8M-like
    # golden largest), against about 0.1 % for fp16
    assert e8 <= 0.15 and r8 <= 0.15


def layer_inputs_and_outputs(model, tok):
    """Every layer's input and output of one fp8 forward: the representations 0 .. N (N after the final LayerNorm)."""
    N = model.num_layers
    return model(tok, repr_layers=list(range(N + 1)))["representations"]


def check_against_emulation(model, tok, name):
    """Each layer of an fp8 forward against the float64 emulation of the same quantisation steps started from that
    layer's input (fp8_refs.emulate_layer; the last layer through the final LayerNorm).  Tolerance: twice the larger
    rel-Fro distance of two perturbed emulations, which carry an error of the full accumulation / rounding bound with
    random signs at every point where the library accumulates or rounds (the GEMM tests measure the library's own
    errors at <= 0.61 of those bounds).  A scale or weight handed to the wrong GEMM moves the output by the e4m3 step
    of every element, an order of magnitude more."""
    reps = layer_inputs_and_outputs(model, tok)
    pad = tok.eq(model.padding_idx)
    N = model.num_layers
    ln = model.emb_layer_norm_after
    for i, layer in enumerate(model.layers):
        rot = layer.self_attn.rot_emb
        inv = rot.inv_freq if rot is not None else None
        runs = [fr.emulate_layer(layer, reps[i], pad, inv, gen=None if k < 0 else torch.Generator().manual_seed(k))
                for k in (-1, 0, 1)]
        if i == N - 1:
            runs = [fr._ln(r, ln.weight.detach().double(), ln.bias.detach().double(), ln.eps)[0] for r in runs]
        emu = runs[0]
        spread = max(rel(r, emu) for r in runs[1:])
        err = rel(reps[i + 1], emu)
        print(f"FP8 emulation {name} layer {i}: rel-Fro lib - emu {err:.2e}, perturbed emulations {spread:.2e}")
        assert math.isfinite(spread) and err <= 2 * spread, (name, i)


@pytest.mark.parametrize("E,H", [(256, 4), (320, 20), (256, 2)], ids=["d64", "d16-partialK", "d128-two-slots"])
def test_layer_against_float64_emulation(E, H):
    """Two fp8 layers whose matrices have block scales several powers of two apart (so that a scale array handed to the
    wrong GEMM, or a weight packed into the wrong slot, moves outputs far outside the bound)."""
    model = build(2, E, H, seed=E + H)
    g = torch.Generator().manual_seed(E * H)
    with torch.no_grad():
        for layer in model.layers:
            for lin, gain in ((layer.self_attn.q_proj, 0.5), (layer.self_attn.k_proj, 2.0),
                              (layer.self_attn.v_proj, 1.0), (layer.fc1, 4.0), (layer.fc2, 0.25)):
                rows = torch.exp(0.7 * torch.randn(lin.weight.shape[0], 1, generator=g)).cuda()
                lin.weight.mul_(gain * rows)
    model.set_precision("fp8")
    tok = torch.randint(4, 24, (3, 200), generator=g)
    tok[:, 0], tok[:, -1] = 0, 2
    tok[1, 150:] = 1
    tok[1, 149] = 2
    check_against_emulation(model, tok.cuda(), f"layer E={E} H={H}")


def test_contacts_in_fp8():
    model = build(2, 128, 2, seed=3)
    model.set_precision("fp8")
    g = torch.Generator().manual_seed(5)
    tok = torch.randint(4, 24, (3, 90), generator=g)
    tok[:, 0], tok[:, -1] = 0, 2
    tok[2, 60:] = 1
    tok[2, 59] = 2
    tok = tok.cuda()
    out = model(tok, return_contacts=True)
    ref = model.contact_head(tok, out["attentions"])
    assert torch.allclose(out["contacts"], ref, rtol=1e-5, atol=1e-6)


def test_variant_scorers_in_fp8():
    """masked_marginals / wt_marginals in fp8 (LM head rows through _lm_head_rows) are bit-identical to the forward on
    each masked copy (resp. the sequence), read at the masked row."""
    from esm_b200 import variants
    model = build(2, 128, 2, seed=4)
    model.set_precision("fp8")
    g = torch.Generator().manual_seed(6)
    tok = torch.randint(4, 24, (1, 70), generator=g)
    tok[:, 0], tok[:, -1] = 0, 2
    tok = tok.cuda()
    pos = [1, 17, 40, 68]
    mm = variants.masked_marginals(model, tok, pos)
    for k, p in enumerate(pos):
        copy = tok.clone()
        copy[0, p] = model.mask_idx
        ref = variants.log_softmax_rows(model(copy)["logits"][0, p:p + 1].contiguous())
        assert torch.equal(mm[k:k + 1], ref)
    wt = variants.wt_marginals(model, tok)
    assert torch.equal(wt, variants.log_softmax_rows(model(tok)["logits"][0].contiguous()))
