"""GPU (-m gpu): the fp32x3 precision of the MSA Transformer (MSATransformer.set_precision("fp32x3")): every MMA operand of
the axial stack is an fp16 hi | lo pair.

  * the split tied row attention and the split column attention kernels against float64 torch;
  * the axial layer and the whole model against the reference's goldens, and 12 layers at MSA-1b width against the
    oracle run in float64;
  * masked-marginal scores of a 12-layer model against the reference's eager fp32;
  * determinism, switching back to fp16, mixed-precision stacks, and predict_cli --precision.

Every comparison prints a PARITY line. Padding positions are not compared, as in test_gpu_msa.py."""
import argparse
import csv
import io
import json
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # variant_fixtures

import test_gpu_tied_attention as tied  # noqa: E402
from test_gpu_msa import assert_maps_change_no_bit, col_maps_against_oracle  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")


def rel_fro(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm())


def max_abs(a, b):
    return float((torch.as_tensor(a).double() - torch.as_tensor(b).double()).abs().max())


def _ptr(t):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def split16(x):
    """fp32 [..., n] -> fp16 hi, lo with hi + lo = x to ~22 bits."""
    hi = x.half()
    return hi, (x - hi.float()).half()


def join16(hi_lo, n):
    return hi_lo[..., :n].float() + hi_lo[..., n:].float()


# ---- kernels ----------------------------------------------------------------------------------------------------
def tied_inputs(B, R, C, H, sharp, seed):
    """q, k, v fp32 [B,R,C,H,64] (q pre-scaled so that the summed logits have std `sharp`) and key_pad [B,C]."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, R, C, H, 64, device="cuda", generator=g) * (sharp / (R * 64) ** 0.5)
    k = torch.randn(B, R, C, H, 64, device="cuda", generator=g)
    v = torch.randn(B, R, C, H, 64, device="cuda", generator=g)
    pad = torch.zeros(B, C, dtype=torch.bool, device="cuda")
    pad[:, C - max(1, C // 9):] = True            # trailing padded key columns
    pad[0, C // 3] = True                          # and one inside
    q = q * (~pad)[:, None, :, None, None]         # q is zeroed at padded positions (axial_attention.py:82-85)
    return q, k, v, pad


def tied_torch(q, k, v, pad, dtype):
    logits = torch.einsum("brihd,brjhd->hbij", q.to(dtype), k.to(dtype))
    logits = logits.masked_fill(pad[None, :, None, :], -10000)
    probs = logits.softmax(-1)
    return torch.einsum("hbij,brjhd->brihd", probs, v.to(dtype)), probs


def run_tied(q, k, v, pad, split):
    from esm_b200 import _lib
    lib = _lib.load()
    B, R, C, H, d = q.shape
    E = H * d
    M = B * R * C
    qkv32 = torch.cat([t.reshape(M, E) for t in (q, k, v)], 1)
    if split:
        qkv = torch.cat(split16(qkv32), 1).contiguous()
        nbytes, fn = lib.esmb200_tied_row_attention_split_scratch_bytes(B, C, H), lib.esmb200_tied_row_attention_split
    else:
        qkv = qkv32.half().contiguous()
        nbytes, fn = lib.esmb200_tied_row_attention_scratch_bytes(B, C, H), lib.esmb200_tied_row_attention
    ctx = torch.empty((M, (2 if split else 1) * E), dtype=torch.float16, device="cuda")
    probs = torch.empty((H, B, C, C), dtype=torch.float32, device="cuda")
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    key_pad = pad.to(torch.uint8).contiguous()
    _lib.check(fn(_ptr(qkv), _ptr(key_pad), _ptr(ctx), _ptr(probs), B, R, C, H, _ptr(scratch), nbytes, _stream()))
    out = join16(ctx, E) if split else ctx.float()
    return out.view(B, R, C, H, d), probs


@pytest.mark.parametrize("B,R,C,H", [(2, 64, 130, 4), (1, 5, 300, 2), (1, 1024, 64, 2)])
def test_split_tied_row_attention_against_float64(B, R, C, H):
    """Sharp logits (std 8 after the sum over R*64 products) with key padding. At R = 1024 the logits are sums of
    65,536 products: the split kernel adds each alignment row's 64-wide slab into the running sum in fp32.  Every stage
    is held to its float64 bound by test_gpu_tied_attention.check_tied; the PARITY line also gives torch's fp32 and the
    fp16 entry point on the same inputs."""
    torch.backends.cuda.matmul.allow_tf32 = False
    q, k, v, pad = tied_inputs(B, R, C, H, sharp=8.0, seed=B * 1000 + R + C)
    want, pwant = tied_torch(q, k, v, pad, torch.float64)
    f32, p32 = tied_torch(q, k, v, pad, torch.float32)
    qkv = tied.pack(torch.stack([q, k, v], 3), True)
    key_pad = pad.to(torch.uint8).contiguous()
    ctx, pgot = tied.check_tied("msa_precision sharp", qkv, key_pad, B, R, C, H, True)
    got = join16(ctx, H * 64).float().view(B, R, C, H, 64)
    g16, p16 = run_tied(q, k, v, pad, False)
    keep = ~pad[:, None, :].expand(B, R, C)       # query positions that are not padding
    r, m = rel_fro(got[keep], want[keep]), max_abs(pgot, pwant)
    print(f"PARITY msa_precision tied_row (B,R,C,H)=({B},{R},{C},{H}): fp32x3 ctx rel_fro={r:.3e} probs max_abs={m:.3e}"
          f"; torch fp32 {rel_fro(f32[keep], want[keep]):.3e} / {max_abs(p32, pwant):.3e}"
          f"; fp16 entry point {rel_fro(g16[keep], want[keep]):.3e} / {max_abs(p16, pwant):.3e}", flush=True)
    assert r <= 2e-5 and m <= 5e-5


def column_inputs(B, R, C, H, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(B, R, C, H, 64, device="cuda", generator=g) * (3.0 / 8.0)   # logits with std 3
    k = torch.randn(B, R, C, H, 64, device="cuda", generator=g)
    v = torch.randn(B, R, C, H, 64, device="cuda", generator=g)
    pad = torch.zeros(B, R, C, dtype=torch.bool, device="cuda")
    pad[:, :, C - 2:] = True                       # trailing padded columns (every row)
    pad[B - 1, R - R // 4:] = True                 # trailing padded rows of the last alignment
    return q, k, v, pad


@pytest.mark.parametrize("B,R,C,H", [(2, 37, 20, 2), (1, 150, 9, 4)])
def test_split_column_attention_against_float64(B, R, C, H):
    """esmb200_column_attention_split reads the row-major [B*R*C, 6E] qkv with strided boxes (6E per column); the
    reference is torch float64 on the column-regrouped tensor. Fully padded columns are not compared."""
    from esm_b200 import _lib
    lib = _lib.load()
    q, k, v, pad = column_inputs(B, R, C, H, seed=R * 10 + C)
    E = H * 64
    M = B * R * C
    # float64 reference, per column: [B, C, H, R, R]
    qt, kt, vt = (t.double().permute(0, 2, 3, 1, 4) for t in (q, k, v))      # [B, C, H, R, 64]
    logits = qt @ kt.transpose(-1, -2)
    logits = logits.masked_fill(pad.permute(0, 2, 1)[:, :, None, None, :], float("-inf"))
    probs = torch.nan_to_num(logits.softmax(-1), nan=0.0)
    want = (probs @ vt).permute(0, 3, 1, 2, 4)                                # [B, R, C, H, 64]
    qkv = torch.cat(split16(torch.cat([t.reshape(M, E) for t in (q, k, v)], 1)), 1).contiguous()
    ctx = torch.empty((M, 2 * E), dtype=torch.float16, device="cuda")
    col_pad = pad.permute(0, 2, 1).contiguous().to(torch.uint8)
    scratch = torch.empty(lib.esmb200_attention_scratch_bytes(B * C, R), dtype=torch.uint8, device="cuda")
    _lib.check(lib.esmb200_column_attention_split(_ptr(qkv), _ptr(col_pad), _ptr(ctx), B, R, C, H, _ptr(scratch),
                                                  _stream()))
    got = join16(ctx, E).view(B, R, C, H, 64)
    keep = ~pad
    r = rel_fro(got[keep], want[keep])
    print(f"PARITY msa_precision column (B,R,C,H)=({B},{R},{C},{H}): fp32x3 ctx rel_fro={r:.3e}", flush=True)
    assert r <= 1e-5


# ---- the axial layer and the model --------------------------------------------------------------------------------
def build_layer(E, Fd, H, precision="fp32x3"):
    from esm_b200.msa import AxialTransformerLayer
    from oracle.msa_oracle import make_axial_state_dict
    sd = make_axial_state_dict(E, Fd, seed=0)
    layer = AxialTransformerLayer(E, Fd, H)
    layer.load_state_dict({k[len("layers.0."):]: v for k, v in sd.items()}, strict=True)
    layer.precision = {"fp16": 0, "fp32x3": 1}[precision]
    return layer.eval().cuda()


@pytest.mark.parametrize("name", ["msa_mid_E256_H4", "msa_small_E128_H2"])
def test_axial_layer_fp32x3_against_reference_golden(name, golden_dir):
    fx = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    cfg, mask = fx["config"], fx["mask"]
    g = torch.Generator().manual_seed(cfg["x_seed"])
    x = torch.randn(cfg["B"], cfg["R"], cfg["C"], cfg["E"], generator=g)
    layer = build_layer(cfg["E"], cfg["F"], cfg["H"])
    keep = torch.ones(x.shape[:3], dtype=torch.bool) if mask is None else ~mask
    kw = {} if mask is None else {"self_attn_padding_mask": mask.cuda()}
    outs = []
    for need in (False, True):
        res = layer(x.permute(1, 2, 0, 3).cuda(), need_head_weights=need, **kw)
        out = (res[0] if need else res).permute(2, 0, 1, 3).cpu()
        outs.append(out)
        r = rel_fro(out[keep], fx["out"][keep])
        line = f"PARITY msa_precision axial_layer {name} maps={need}: out rel_fro={r:.3e}"
        assert r <= 2e-5, line
        if need:
            mr = max_abs(res[2].cpu(), fx["row_attn"])
            col = res[1][:, :4].cpu()                                # [H, 4 columns, B, R, R]
            qkeep = keep[:, :, :4].permute(2, 0, 1)                  # [4, B, R]
            mc = float((col - fx["col_attn_sample"]).abs()[:, qkeep].max())
            line += f" row maps max_abs={mr:.3e} column sample max_abs={mc:.3e}"
            assert mr <= 5e-5 and mc <= 5e-5, line
        print(line, flush=True)
    assert torch.equal(outs[0], outs[1])  # the maps change no bit of x


def build_model(cfg, seed=None):
    from esm_b200.msa import MSATransformer
    from oracle.msa_oracle import make_msa_state_dict
    sd = make_msa_state_dict(cfg["layers"], cfg["E"], cfg["F"], cfg["H"], seed=cfg["seed"] if seed is None else seed)
    model = MSATransformer(argparse.Namespace(layers=cfg["layers"], embed_dim=cfg["E"], ffn_embed_dim=cfg["F"],
                                              attention_heads=cfg["H"], max_positions=1024, embed_positions_msa=True))
    model.load_state_dict(sd, strict=True)
    return model.eval().cuda(), sd


@pytest.mark.parametrize("name", ["msa_model_L2_E128_H2", "msa_model_L3_E256_H4_nopad"])
def test_msa_transformer_fp32x3_against_reference_golden(name, golden_dir):
    fx = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    cfg, tokens = fx["config"], fx["tokens"]
    model, sd = build_model(cfg)
    model.set_precision("fp32x3")
    keep = tokens.ne(1)
    L = cfg["layers"]
    out = model(tokens.cuda(), repr_layers=[0, 1, L], return_contacts=True)
    assert_maps_change_no_bit(model, tokens.cuda(), out, [0, 1, L])
    reprs = {k: rel_fro(out["representations"][k].cpu()[keep], v[keep]) for k, v in fx["representations"].items()}
    lg = rel_fro(out["logits"].cpu()[keep], fx["logits"][keep])
    ra = max_abs(out["row_attentions"].cpu(), fx["row_attentions"])
    ct = max_abs(out["contacts"].cpu(), fx["contacts"])
    pc = max_abs(model.predict_contacts(tokens.cuda()).cpu(), fx["contacts"])    # no column maps
    out3 = model(tokens.cuda(), need_head_weights=True)
    col = out3["col_attentions"][:, :, :, :3].cpu()
    qkeep = keep[:, :, :3].permute(0, 2, 1)                                     # [B, 3, R]
    cs = float((col - fx["col_attentions_sample"]).abs().permute(0, 3, 4, 1, 2, 5)[qkeep].max())
    ra3 = max_abs(out3["row_attentions"].cpu(), fx["row_attentions"])
    c64 = col_maps_against_oracle(f"msa_precision model {name} fp32x3", sd, cfg, tokens, out3["col_attentions"])
    print(f"PARITY msa_precision model {name}: repr rel_fro {', '.join(f'{k}:{v:.3e}' for k, v in reprs.items())}; "
          f"logits rel_fro={lg:.3e}; row maps max_abs={ra:.3e} (need_head_weights {ra3:.3e}); column sample "
          f"max_abs={cs:.3e}; contacts max_abs={ct:.3e} (predict_contacts {pc:.3e})", flush=True)
    assert all(v <= 2e-5 for v in reprs.values()) and lg <= 2e-5
    assert ra <= 5e-5 and ra3 <= 5e-5 and cs <= 5e-5 and c64 <= 5e-5
    assert ct <= 1e-4 and pc <= 1e-4


def test_twelve_layers_msa1b_width_against_float64_oracle():
    """12 layers at esm_msa1b width (E=768, H=12, F=3072), two padded MSAs of 32 x 256, against the oracle run in
    float64 on the device; the fp16 figure of the same model is printed beside it."""
    from oracle import msa_oracle
    cfg = dict(layers=12, E=768, F=3072, H=12, seed=3)
    model, sd = build_model(cfg)
    tokens = msa_oracle.make_msa_tokens(2, 32, 256, seed=21, pad_cols=19, pad_rows_last=6)
    keep = tokens.ne(1)
    ref = msa_oracle.msa_transformer_forward({k: v.double().cuda() for k, v in sd.items()}, 12, 12, tokens.cuda(),
                                             repr_layers=[12])
    want_r, want_l = ref["representations"][12].cpu(), ref["logits"].cpu()
    del ref
    res = {}
    for prec in ("fp16", "fp32x3"):
        model.set_precision(prec)
        out = model(tokens.cuda(), repr_layers=[12])
        res[prec] = (rel_fro(out["representations"][12].cpu()[keep], want_r[keep]),
                     rel_fro(out["logits"].cpu()[keep], want_l[keep]))
    print(f"PARITY msa_precision 12 layers E=768 2x32x256 padded vs float64 oracle: fp32x3 repr rel_fro="
          f"{res['fp32x3'][0]:.3e} logits {res['fp32x3'][1]:.3e}; fp16 repr {res['fp16'][0]:.3e} logits "
          f"{res['fp16'][1]:.3e}", flush=True)
    assert max(res["fp32x3"]) <= 1e-4
    assert max(res["fp32x3"]) * 10 <= min(res["fp16"])


def _centered_rel_fro(got, want):
    got = got.double() - got.double().mean(-1, keepdim=True)
    want = want.double() - want.double().mean(-1, keepdim=True)
    return float((got - want).norm() / want.norm())


def test_masked_marginals_fp32x3_against_the_reference():
    """The setup of test_gpu_variants.py's MSA test: 12 layers at MSA-1b width, an unpadded 64 x 100 alignment, 16
    masked columns, against the unmodified reference in eager fp32 (TF32 off)."""
    if not os.path.isdir(os.path.join(REF, "esm")):
        pytest.fail("oracle/_ref/esm is missing: build() copies the reference there (oracle/reference.py)")
    from esm_b200 import MSATransformer, variants
    from oracle.msa_oracle import make_msa_state_dict, make_msa_tokens
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    L, E, Fd, H = 12, 768, 3072, 12
    args = argparse.Namespace(layers=L, embed_dim=E, ffn_embed_dim=Fd, attention_heads=H, dropout=0.0,
                              attention_dropout=0.0, activation_dropout=0.0, max_tokens_per_msa=2 ** 14,
                              max_tokens=2 ** 14, max_positions=1024, embed_positions_msa=True)
    sd = make_msa_state_dict(L, E, Fd, H, seed=0)
    tokens = make_msa_tokens(1, 64, 101, seed=7)
    positions = list(range(0, 101, 7))[:16]
    sys.path.insert(0, REF)
    try:
        import esm as esm_ref
        ref = esm_ref.MSATransformer(args, esm_ref.Alphabet.from_architecture("msa_transformer"))
    finally:
        sys.path.remove(REF)
    ref.load_state_dict(sd, strict=True)
    ref = ref.eval().cuda()
    rows = []
    with torch.no_grad():
        for i in positions:  # predict.py:170-177
            masked = tokens.clone()
            masked[0, 0, i] = ref.mask_idx
            rows.append(torch.log_softmax(ref(masked.cuda())["logits"], dim=-1)[:, 0, i])
    want = torch.cat(rows).cpu()
    del ref
    torch.cuda.empty_cache()
    model = MSATransformer(args, "msa_transformer")
    model.load_state_dict(sd, strict=True)
    model = model.eval().cuda()
    r16 = _centered_rel_fro(variants.masked_marginals(model, tokens, positions=positions).cpu(), want)
    model.set_precision("fp32x3")
    r32 = _centered_rel_fro(variants.masked_marginals(model, tokens, positions=positions).cpu(), want)
    print(f"PARITY msa_precision masked-marginals 12 layers 64x100 vs reference eager fp32: fp32x3 centered "
          f"rel_fro={r32:.3e}, fp16 {r16:.3e} ({r16 / r32:.1f}x)", flush=True)
    assert r32 <= 1e-3 and r32 * 10 <= r16


# ---- behaviour ----------------------------------------------------------------------------------------------------
def test_fp32x3_is_deterministic(golden_dir):
    fx = torch.load(os.path.join(golden_dir, "msa_model_L2_E128_H2.pt"), weights_only=False)
    model, _ = build_model(fx["config"])
    model.set_precision("fp32x3")
    tokens = fx["tokens"].cuda()
    for kw in ({}, {"need_head_weights": True}, {"return_contacts": True}):
        a, b = model(tokens, repr_layers=[2], **kw), model(tokens, repr_layers=[2], **kw)
        for key in a:
            if key == "representations":
                assert torch.equal(a[key][2], b[key][2]), kw
            else:
                assert torch.equal(a[key], b[key]), (kw, key)
    print("PARITY msa_precision determinism: two fp32x3 calls bit-identical with and without maps", flush=True)


def test_switching_back_to_fp16_is_bit_identical(golden_dir):
    fx = torch.load(os.path.join(golden_dir, "msa_model_L2_E128_H2.pt"), weights_only=False)
    tokens = fx["tokens"].cuda()
    never, _ = build_model(fx["config"])
    switched, _ = build_model(fx["config"])
    switched.set_precision("fp32x3")
    s32 = switched(tokens, repr_layers=[2], return_contacts=True)
    switched.set_precision("fp16")
    for kw in ({"return_contacts": True}, {"need_head_weights": True}, {}):
        a, b = never(tokens, repr_layers=[2], **kw), switched(tokens, repr_layers=[2], **kw)
        assert torch.equal(a["logits"], b["logits"]) and torch.equal(a["representations"][2], b["representations"][2])
        for key in ("row_attentions", "col_attentions", "contacts"):
            if key in a:
                assert torch.equal(a[key], b[key]), (kw, key)
    assert not torch.equal(s32["logits"], never(tokens)["logits"])  # the fp32x3 pass did run in the other mode
    print("PARITY msa_precision fp32x3 -> fp16: bit-identical to a model that was never switched", flush=True)


def test_mixed_precision_stack_is_rejected():
    from esm_b200 import _lib
    from esm_b200.msa import run_axial_stack
    l16, l32 = build_layer(128, 512, 2, "fp16"), build_layer(128, 512, 2, "fp32x3")
    x = torch.randn(1, 4, 40, 128, device="cuda")
    for layers in ([l16, l32], [l32, l16]):
        with pytest.raises(_lib.Esmb200Error, match="share one precision"):
            run_axial_stack(layers, x.clone())
    # a fp16 row layer with a fp32x3 column layer inside one AxialTransformerLayer
    lib = _lib.load()
    row16 = l16.handles()[0]
    col32 = l32.handles()[1]
    import ctypes
    nbytes = lib.esmb200_axial_workspace_bytes_split(128, 512, 1, 4, 40)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    rc = lib.esmb200_axial_stack_forward((ctypes.c_void_p * 1)(row16), (ctypes.c_void_p * 1)(col32), 1, _ptr(x), None,
                                         None, 1, 4, 40, None, None, _ptr(ws), nbytes, _stream())
    assert rc == -1 and b"share one precision" in lib.esmb200_last_error()


# ---- the command line -----------------------------------------------------------------------------------------------
def test_predict_cli_fp32x3_is_closer_to_predict_py(golden_dir, tmp_path):
    import variant_fixtures as vf
    from esm_b200 import predict_cli
    with open(os.path.join(golden_dir, "variants.json")) as f:
        fixture = json.load(f)
    (tmp_path / "dms.csv").write_text(fixture["dms_csv"])
    (tmp_path / "msa.a3m").write_text(fixture["a3m"])
    names = ["esm2_t2_tiny", "msa_t2_tiny"]
    paths = [vf.write_checkpoint(n, vf.MODELS[n], str(tmp_path)) for n in names]
    cols = {}
    for prec in ("fp16", "fp32x3"):
        out = tmp_path / f"out_{prec}.csv"
        args = predict_cli.create_parser().parse_args(
            ["--model-location"] + paths + ["--sequence", fixture["sequence"], "--dms-input", str(tmp_path / "dms.csv"),
                                            "--dms-output", str(out), "--offset-idx", str(fixture["offset_idx"]),
                                            "--scoring-strategy", "masked-marginals", "--msa-path",
                                            str(tmp_path / "msa.a3m"), "--msa-samples", str(fixture["msa_samples"]),
                                            "--precision", prec])
        predict_cli.run(args)
        got = list(csv.reader(io.StringIO(out.read_text())))
        cols[prec] = [[float(r[4 + j]) for r in got[1:]] for j in range(len(names))]
    for j, n in enumerate(names):
        table = list(csv.reader(io.StringIO(fixture["outputs"][f"{n}/masked-marginals"])))
        want = [float(r[-1]) for r in table[1:]]
        r16, r32 = rel_fro(cols["fp16"][j], want), rel_fro(cols["fp32x3"][j], want)
        print(f"PARITY msa_precision predict_cli {n} masked-marginals: fp32x3 rel_fro={r32:.3e}, fp16 {r16:.3e}",
              flush=True)
        assert r32 < r16
