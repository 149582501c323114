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


quantize_dev = fr.quantize_dev


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


M_ALL = [1, 127, 128, 129, 4097]
CASES = ([("650M", "fc1", M) for M in M_ALL] + [("650M", "fc2", M) for M in M_ALL] + [("650M", "qkv", M) for M in M_ALL]
         + [(m, p, 129) for m in MODELS for p in ("qkv", "fc1", "fc2")]
         + [(m, p, 4097) for m in ("8M", "35M", "15B") for p in ("qkv", "fc1", "fc2")])


EPIS = {"qkv": 0, "fc2": 1, "fc1": 5}  # EPI_QKV_ROPE (fp16 out, rope), EPI_BIAS_RESIDUAL (x += y), EPI_GELU_FP8


KIND_CASES = [c + (k,) for c in CASES for k in ("gauss", "spread")]


@pytest.mark.parametrize("model,proj,M,kind", KIND_CASES,
                         ids=[f"{m}-{p}-{M}" + ("-spread" if k == "spread" else "") for m, p, M, k in KIND_CASES])
def test_gemm_fp8(model, proj, M, kind):
    """Every model's (N, K) of the three projections on Gaussian operands (nearly uniform block scales) and on operands
    whose row, K-block and weight-block scales span many octaves (fp8_refs.spread_operands), so that a scale read from
    the wrong row, K block or weight block moves results by powers of two.  ESM-1b / 1v share 650M's shapes; their
    table-free QKV epilogue runs in tests/test_gpu_stack_isolation.py."""
    N, K = shapes(model)[proj]
    r = fr.check_gemm(EPIS[proj], M, N, K, kind, seed=M * 7 + N + K)
    print(f"PARITY fp8 gemm {kind} {model} {proj} M={M} N={N} K={K}: err/bound={r['ratio']:.3f} "
          f"flips={r['flips']}/{M * N} scale_flips={r['scale_flips']}", flush=True)


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
    errors at <= 0.61 of that size on Gaussian operands).  A scale or weight handed to the wrong GEMM moves the output
    by the e4m3 step of every element, an order of magnitude more."""
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


@pytest.mark.parametrize("E,H", [(256, 4), (320, 20), (256, 2), (480, 20), (384, 4)],
                         ids=["d64", "d16-partialK", "d128-two-slots", "d24", "d96-partial-second-slot"])
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
