"""GPU (-m gpu): the MSA axial block (esm_b200.msa.AxialTransformerLayer -> C ABI -> sm_90a kernels) against the
committed outputs of the reference's AxialTransformerLayer and against the CPU oracle. Same tolerance as the ESM-2
path (fp16 operands): rel-Frobenius <= 3e-3 on the layer output, probabilities max-abs <= 1e-2."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_fro(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def build(E, Fd, H, seed=0):
    from esm_b200.msa import AxialTransformerLayer
    from oracle.msa_oracle import make_axial_state_dict
    sd = make_axial_state_dict(E, Fd, seed=seed)
    layer = AxialTransformerLayer(E, Fd, H)
    layer.load_state_dict({k[len("layers.0."):]: v for k, v in sd.items()}, strict=True)
    return layer.eval().cuda(), sd


def test_axial_layer_against_reference_golden(golden_dir):
    fx = torch.load(os.path.join(golden_dir, "msa_mid_E256_H4.pt"), weights_only=False)
    cfg = fx["config"]
    g = torch.Generator().manual_seed(cfg["x_seed"])
    x = torch.randn(cfg["B"], cfg["R"], cfg["C"], cfg["E"], generator=g)
    layer, _ = build(cfg["E"], cfg["F"], cfg["H"])
    out, col, row = layer(x.permute(1, 2, 0, 3).cuda(), need_head_weights=True)  # reference layout (R,C,B,E)
    assert out.shape == (cfg["R"], cfg["C"], cfg["B"], cfg["E"])
    assert torch.equal(out, layer(x.permute(1, 2, 0, 3).cuda()))  # the maps change no bit of x
    assert rel_fro(out.permute(2, 0, 1, 3).cpu(), fx["out"]) <= 3e-3
    assert row.shape == fx["row_attn"].shape
    assert float((row.cpu() - fx["row_attn"]).abs().max()) <= 1e-2
    assert float((col[:, :4].cpu() - fx["col_attn_sample"]).abs().max()) <= 1e-2


def test_axial_layer_against_oracle_msa1b_width():
    """esm_msa1b width (E=768, H=12, F=3072), 2 MSAs of 16 rows x 192 columns."""
    from oracle import msa_oracle
    layer, sd = build(768, 3072, 12)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 16, 192, 768, generator=g)
    ref = msa_oracle.axial_layer(x, sd, "layers.0.", 12)
    out = layer(x.permute(1, 2, 0, 3).cuda())
    assert rel_fro(out.permute(2, 0, 1, 3).cpu(), ref) <= 3e-3


def test_padded_msas_against_reference_golden(golden_dir):
    """Two MSAs padded the way MSABatchConverter pads (trailing columns; trailing rows of the second MSA): q zeroing,
    -10000 key fill in the row attention, padded keys in the column attention. Padding positions themselves are not
    compared (fully padded columns: the reference averages v uniformly, this path writes 0 — documented deviation)."""
    fx = torch.load(os.path.join(golden_dir, "msa_small_E128_H2.pt"), weights_only=False)
    cfg, mask = fx["config"], fx["mask"]
    g = torch.Generator().manual_seed(cfg["x_seed"])
    x = torch.randn(cfg["B"], cfg["R"], cfg["C"], cfg["E"], generator=g)
    layer, _ = build(cfg["E"], cfg["F"], cfg["H"])
    keep = ~mask
    outs = []
    for need in (False, True):
        res = layer(x.permute(1, 2, 0, 3).cuda(), self_attn_padding_mask=mask.cuda(), need_head_weights=need)
        out = (res[0] if need else res).permute(2, 0, 1, 3).cpu()
        outs.append(out)
        assert torch.isfinite(out).all()
        assert rel_fro(out[keep], fx["out"][keep]) <= 3e-3
        if need:
            assert float((res[2].cpu() - fx["row_attn"]).abs().max()) <= 1e-2
            col = res[1][:, :4].cpu()                       # [H, 4 columns, B, R, R]; columns 0-3 are not padding
            qkeep = keep[:, :, :4].permute(2, 0, 1)         # [4, B, R]: query rows that are not padding
            assert float((col - fx["col_attn_sample"]).abs()[:, qkeep].max()) <= 1e-2
    assert torch.equal(outs[0], outs[1])  # the maps change no bit of x


@pytest.mark.parametrize("B,R,C", [(1, 10, 77), (2, 5, 130), (1, 3, 300), (1, 130, 40)])
def test_axial_layer_ragged_shapes_against_oracle(B, R, C):
    """Row counts that are not a multiple of the 4-row update tile (and > 128: two query tiles in the column attention),
    column counts that are not multiples of 64 / 4."""
    from oracle import msa_oracle
    layer, sd = build(128, 512, 2)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(B, R, C, 128, generator=g)
    ref, col_ref, row_ref = msa_oracle.axial_layer(x, sd, "layers.0.", 2, need_head_weights=True)
    out = layer(x.permute(1, 2, 0, 3).cuda())
    assert rel_fro(out.permute(2, 0, 1, 3).cpu(), ref) <= 3e-3
    out2, col, row = layer(x.permute(1, 2, 0, 3).cuda(), need_head_weights=True)
    assert rel_fro(out2.permute(2, 0, 1, 3).cpu(), ref) <= 3e-3
    assert float((row.cpu() - row_ref).abs().max()) <= 1e-2
    assert float((col.cpu() - col_ref).abs().max()) <= 1e-2


def build_model(cfg):
    from argparse import Namespace
    from esm_b200.msa import MSATransformer
    from oracle.msa_oracle import make_msa_state_dict
    sd = make_msa_state_dict(cfg["layers"], cfg["E"], cfg["F"], cfg["H"], seed=cfg["seed"])
    model = MSATransformer(Namespace(layers=cfg["layers"], embed_dim=cfg["E"], ffn_embed_dim=cfg["F"],
                                     attention_heads=cfg["H"], max_positions=1024, embed_positions_msa=True))
    model.load_state_dict(sd, strict=True)
    return model.eval().cuda(), sd


def assert_maps_change_no_bit(model, tokens, out, repr_layers):
    """out = model(tokens, repr_layers, return_contacts=True), with the column maps: the same call without them, and
    predict_contacts, give the same bits (one stack call computes every map)"""
    model.contacts_without_col_attentions = True
    lean = model(tokens, repr_layers=repr_layers, return_contacts=True)
    model.contacts_without_col_attentions = False
    assert "col_attentions" not in lean
    for key in ("logits", "row_attentions", "contacts"):
        assert torch.equal(lean[key], out[key]), key
    for k in repr_layers:
        assert torch.equal(lean["representations"][k], out["representations"][k]), k
    assert torch.equal(model.predict_contacts(tokens), out["contacts"])


@pytest.mark.parametrize("name", ["msa_model_L2_E128_H2", "msa_model_L3_E256_H4_nopad"])
def test_msa_transformer_against_reference_golden(name, golden_dir):
    """esm_b200.msa.MSATransformer (embedding prologue kernel, esmb200_axial_stack_forward, LM head, contact head)
    against the reference's MSATransformer outputs; padding positions are not compared (see msa.py)."""
    fx = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    cfg, tokens = fx["config"], fx["tokens"]
    model, sd = build_model(cfg)
    keep = tokens.ne(1)
    L = cfg["layers"]
    out = model(tokens.cuda(), repr_layers=[0, 1, L], return_contacts=True)
    assert "col_attentions" in out  # return_contacts implies need_head_weights (msa_transformer.py:149-150)
    assert_maps_change_no_bit(model, tokens.cuda(), out, [0, 1, L])
    for k, v in fx["representations"].items():
        assert rel_fro(out["representations"][k].cpu()[keep], v[keep]) <= (1e-5 if k == 0 else 3e-3), k
    assert rel_fro(out["logits"].cpu()[keep], fx["logits"][keep]) <= 4e-3
    assert float((out["row_attentions"].cpu() - fx["row_attentions"]).abs().max()) <= 1e-2
    assert float((out["contacts"].cpu() - fx["contacts"]).abs().max()) <= 1e-2
    # plain forward (no attention maps): one esmb200_axial_stack_forward call for the whole stack
    out2 = model(tokens.cuda(), repr_layers=[L])
    assert set(out2.keys()) == {"logits", "representations"}
    assert rel_fro(out2["representations"][L].cpu()[keep], fx["representations"][L][keep]) <= 3e-3
    # need_head_weights: column maps too, B x L x H x C x R x R
    out3 = model(tokens.cuda(), need_head_weights=True)
    assert torch.equal(out3["logits"], out2["logits"])
    col = out3["col_attentions"][:, :, :, :3].cpu()
    qkeep = keep[:, :, :3].permute(0, 2, 1)                      # [B, 3, R] query rows that are not padding
    diff = (col - fx["col_attentions_sample"]).abs()             # [B, L, H, 3, R, R]
    assert float(diff.permute(0, 3, 4, 1, 2, 5)[qkeep].max()) <= 1e-2
    assert float((out3["row_attentions"].cpu() - fx["row_attentions"]).abs().max()) <= 1e-2
    # every column map against the oracle in float64, within the row maps' 1e-2
    assert col_maps_against_oracle(f"msa model {name} fp16", sd, cfg, tokens, out3["col_attentions"]) <= 1e-2


def col_maps_against_oracle(name, sd, cfg, tokens, col):
    """max-abs of the column maps col [B,L,H,C,R,R] against oracle.msa_oracle.msa_transformer_forward in float64 over
    every column with a valid key, padded query rows included (the column attention masks keys only); the columns of
    padding only are exactly 0 (the reference gives 1/R there)"""
    from oracle import msa_oracle
    ref = msa_oracle.msa_transformer_forward({k: v.double().cuda() for k, v in sd.items()}, cfg["layers"], cfg["H"],
                                             tokens.cuda(), need_head_weights=True)["col_attentions"]
    live = tokens.ne(1).any(1).cuda()                              # [B, C]
    got = col.permute(0, 3, 1, 2, 4, 5)                            # [B, C, L, H, R, R]
    assert bool((got[~live] == 0).all()), "a column of padding only is not 0"
    m = float((got.double() - ref.permute(0, 3, 1, 2, 4, 5)).abs()[live].max())
    print(f"PARITY {name} column maps vs float64 oracle: max_abs={m:.3e} over {int(live.sum())} live columns",
          flush=True)
    return m


def test_msa_factory_and_batch_converter_end_to_end():
    """esm_b200.pretrained.esm_msa1b_t12_100M_UR50S() -> (model, alphabet) like the reference's factory; a small MSA
    through the batch converter; contacts [B, C-1, C-1] symmetric in (0, 1)."""
    from esm_b200 import pretrained
    model, alphabet = pretrained.esm_msa1b_t12_100M_UR50S(allow_random_init=True)
    model = model.cuda()
    msa = [("s%d" % i, "MKTVRQERLKSIVRILERSKEPVSGAQLAEELSVSRQVIVQDIAYLRSLGYNIVATPRGYVLAGG"[:40]) for i in range(6)]
    _, _, tokens = alphabet.get_batch_converter()(msa)
    assert tokens.shape == (1, 6, 41)
    contacts = model.predict_contacts(tokens.cuda())
    assert contacts.shape == (1, 40, 40)
    assert torch.isfinite(contacts).all() and float(contacts.min()) >= 0 and float(contacts.max()) <= 1
    assert float((contacts - contacts.transpose(1, 2)).abs().max()) <= 1e-6


def test_axial_stack_is_deterministic():
    """Repeated esmb200_axial_stack_forward calls on the same input give the same bits (no atomics on the data path
    except the residual reduce-add, whose per-element order is fixed)."""
    from esm_b200.msa import run_axial_stack
    layer, _ = build(128, 512, 2)
    g = torch.Generator().manual_seed(3)
    x0 = torch.randn(1, 6, 70, 128, generator=g).cuda()
    buf = torch.empty_like(x0)
    outs = []
    for _ in range(4):
        buf.copy_(x0)
        run_axial_stack([layer, layer], buf)
        outs.append(buf.clone())
    torch.cuda.synchronize()
    for o in outs[1:]:
        assert torch.equal(o, outs[0])
    assert torch.isfinite(outs[0]).all()


def test_column_maps_over_the_grid_limit_run_through():
    """Column maps for B*C*H = 66,000 > 65535 (the probability kernel's grid has one z index per map, so the library
    launches it once per 65535 / H column sequences): 33 alignments of one row and 1000 columns.  Every column has one
    key, so every map is exactly 1.0 (the reference's R = 1 case, axial_attention.py:189), and x is the same bits as
    without maps."""
    from esm_b200.msa import run_axial_stack
    layer, _ = build(128, 512, 2)
    x = torch.randn(33, 1, 1000, 128, device="cuda")
    y, z = x.clone(), x.clone()
    col = torch.full((33, 1000, 2, 1, 1), float("nan"), device="cuda")
    run_axial_stack([layer], y, col_attn={0: col})
    run_axial_stack([layer], z)
    torch.cuda.synchronize()
    assert bool((col == 1.0).all())
    assert torch.equal(y, z)
