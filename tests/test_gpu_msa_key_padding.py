"""GPU (-m gpu): per-alignment key padding through the MSA Transformer's axial stack, in fp16 and fp32x3.

A batch of alignments padded the way MSABatchConverter pads (each alignment's own width and depth inside one R x C)
gives alignment b padded key columns of its own.  The stack (esmb200_axial_stack_forward) passes pad_mask [B,R,C] to
the tied row attention at stride R * C, so the keys follow row 0 of each alignment.  Two calls of it are checked,
run_axial_stack with the row maps only and AxialTransformerLayer.forward_batch_major(..., need_probs=True), which also
writes the column maps.  For both:
  * the row-attention probabilities are exactly 0 at each alignment's own padded key columns;
  * each alignment's outputs and row maps at valid positions are bit-identical to that alignment run alone at the
    same R and C;
  * each alignment's column maps, the whole [C,H,R,R] block, are bit-identical to that alignment's run alone;
  * the residual update at valid positions is within the layer tolerances of test_gpu_layer_head_widths (fp16) and
    test_gpu_layer_split (fp32x3) of oracle.msa_oracle.axial_layer in float64, and so are the row maps and the column
    maps at every query row of every column with a valid key (columns of padding only are exactly 0).
A synthetic mask whose row 0 differs from the other rows pins the reference's semantics: padded key columns are those
of row 0, q is zeroed at every padded token.  Two tokenised MSAs of different width and depth go through the whole
MSATransformer against oracle.msa_oracle.msa_transformer_forward in float64."""
import argparse

import pytest
import torch

from test_gpu_layer_head_widths import GATES
from test_gpu_layer_split import LAYER_DELTA_RELFRO, LAYER_PROBS_MAX_ABS

pytestmark = pytest.mark.gpu

E, FD, H = 128, 512, 2
# (rel-Frobenius of the residual update, max-abs of the row maps) at valid positions
TOL = {0: GATES[0], 1: (LAYER_DELTA_RELFRO, LAYER_PROBS_MAX_ABS)}
PRECISIONS = pytest.mark.parametrize("precision", [0, 1], ids=["fp16", "fp32x3"])
PATHS = pytest.mark.parametrize("path", ["stack", "batch_major"])


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def build(precision):
    from esm_b200.msa import AxialTransformerLayer
    from oracle.msa_oracle import make_axial_state_dict
    sd = make_axial_state_dict(E, FD, seed=21)
    layer = AxialTransformerLayer(E, FD, H)
    layer.load_state_dict({k[len("layers.0."):]: v for k, v in sd.items()}, strict=True)
    layer = layer.eval().cuda()
    layer.precision = precision
    return layer, sd


def batch_mask(widths, depths, R, C):
    """[B,R,C] bool: alignment b holds depths[b] rows of widths[b] columns, the rest is padding"""
    pad = torch.ones(len(widths), R, C, dtype=torch.bool)
    for b, (w, d) in enumerate(zip(widths, depths)):
        pad[b, :d, :w] = False
    return pad


def run(layer, x, pad, path):
    """one layer on x [B,R,C,E] -> (out [B,R,C,E], row maps [H,B,C,C], column maps [B,C,H,R,R]) on the CPU; the
    column maps start as NaN, so an entry the call does not write shows"""
    from esm_b200.msa import run_axial_stack
    y = x.clone().cuda()
    B, R, C, _ = x.shape
    if path == "stack":
        col = torch.full((B, C, H, R, R), float("nan"), device="cuda")
        probs = run_axial_stack([layer], y, pad.cuda(), row_attn_layers=[0], col_attn={0: col})[0]
    else:
        probs, col = layer.forward_batch_major(y, pad.cuda(), need_probs=True)
        col = col.permute(2, 1, 0, 3, 4)  # the reference's [H,C,B,R,R] -> [B,C,H,R,R]
    torch.cuda.synchronize()
    return y.cpu(), probs.cpu(), col.cpu()


def against_oracle(name, precision, x, pad, out, probs, sd, col):
    """residual update and row maps at valid positions, and the column maps at every query row of every column with
    a valid key, against the float64 oracle, within TOL"""
    from oracle import msa_oracle
    sd64 = {k: v.double() for k, v in sd.items()}
    ref, cp, rp = msa_oracle.axial_layer(x.double(), sd64, "layers.0.", H, pad, need_head_weights=True)
    keep = ~pad
    d_got, d_ref = (out.double() - x.double())[keep], (ref - x.double())[keep]
    r = float((d_got - d_ref).norm() / d_ref.norm())
    qkeep = ~pad[:, 0]  # [B,C]: query columns that are not padding in row 0
    pa = float((probs.double() - rp).abs()[:, qkeep].max())
    live = keep.any(1)  # [B,C]: columns with a valid key (a column of padding only is 0 here, 1/R in the reference)
    ca = float((col.double() - cp.permute(2, 1, 0, 3, 4)).abs()[live].max())
    assert bool((col[~live] == 0).all()), "a column of padding only is not 0"
    report(name, delta_rel_fro=r, row_maps_max_abs=pa, col_maps_max_abs=ca)
    assert r <= TOL[precision][0] and pa <= TOL[precision][1] and ca <= TOL[precision][1], (r, pa, ca)


@PRECISIONS
@PATHS
def test_alignments_padded_like_the_batch_converter(path, precision):
    B, R, C = 3, 6, 70
    widths, depths = [70, 53, 12], [6, 6, 4]
    layer, sd = build(precision)
    pad = batch_mask(widths, depths, R, C)
    x = torch.randn(B, R, C, E, generator=torch.Generator().manual_seed(7))
    out, probs, col = run(layer, x, pad, path)
    for b, w in enumerate(widths):
        assert bool((probs[:, b, :, w:] == 0).all()), f"alignment {b}: a padded key column has probability"
    bad = bad_col = 0
    for b, w in enumerate(widths):
        ob, pb, cb = run(layer, x[b:b + 1], pad[b:b + 1], path)
        keep = ~pad[b]
        bad += int((out[b][keep] != ob[0][keep]).sum()) + int((probs[:, b, :w] != pb[:, 0, :w]).sum())
        bad_col += int((col[b] != cb[0]).sum())  # the whole [C,H,R,R] block, padded columns and rows included
    report(f"msa key padding {path} precision={precision} alone vs batched", mismatches=float(bad),
           col_map_mismatches=float(bad_col))
    assert bad == 0 and bad_col == 0
    against_oracle(f"msa key padding {path} precision={precision} vs float64", precision, x, pad, out, probs, sd, col)


@PRECISIONS
@PATHS
def test_keys_follow_row_zero(path, precision):
    """Row 0 pads fewer columns than the rows below it: the key columns padded in rows >= 1 only stay attendable,
    their q is zeroed all the same."""
    B, R, C = 2, 5, 70
    pad = torch.zeros(B, R, C, dtype=torch.bool)
    pad[0, 0, 60:] = True
    pad[0, 1:, 50:] = True
    pad[1, 1:, 30:40] = True
    pad[1, 3:] = True
    layer, sd = build(precision)
    x = torch.randn(B, R, C, E, generator=torch.Generator().manual_seed(8))
    out, probs, col = run(layer, x, pad, path)
    assert bool((probs[:, 0, :, 60:] == 0).all()) and bool((probs[:, 0, :60, 50:60] > 0).all())
    assert bool((probs[:, 1, :, 30:40] > 0).all())
    against_oracle(f"msa keys follow row 0 {path} precision={precision}", precision, x, pad, out, probs, sd, col)


@PRECISIONS
def test_msa_transformer_on_a_ragged_batch(precision):
    """Two MSAs of 5 x 40 and 3 x 25 tokens (<cls> included) in one padded batch, against the float64 oracle at the
    valid tokens, with and without need_head_weights."""
    from esm_b200.msa import MSATransformer
    from oracle import msa_oracle
    L = 2
    sd = msa_oracle.make_msa_state_dict(L, E, FD, H, seed=4)
    model = MSATransformer(argparse.Namespace(layers=L, embed_dim=E, ffn_embed_dim=FD, attention_heads=H,
                                              max_positions=1024, embed_positions_msa=True))
    model.load_state_dict(sd, strict=True)
    model = model.eval().cuda()
    if precision:
        model.set_precision("fp32x3")
    tokens = msa_oracle.make_msa_tokens(2, 5, 40, seed=12)
    tokens[1, 3:] = msa_oracle.PAD
    tokens[1, :, 25:] = msa_oracle.PAD
    keep = tokens.ne(msa_oracle.PAD)
    ref = msa_oracle.msa_transformer_forward({k: v.double() for k, v in sd.items()}, L, H, tokens, repr_layers=[L],
                                             need_head_weights=True)
    tol = (3e-3, 4e-3, 1e-2) if precision == 0 else (2e-5, 2e-5, 5e-5)  # test_gpu_msa / test_gpu_msa_precision
    outs = []
    for need in (False, True):
        out = model(tokens.cuda(), repr_layers=[L], need_head_weights=need)
        outs.append(out)
        rep = out["representations"][L].cpu().double()[keep]
        want = ref["representations"][L][keep]
        r = float((rep - want).norm() / want.norm())
        lg = out["logits"].cpu().double()[keep]
        lr = float((lg - ref["logits"][keep]).norm() / ref["logits"][keep].norm())
        ra = float((out["row_attentions"].cpu().double() - ref["row_attentions"]).abs().max()) if need else 0.0
        ca = 0.0
        if need:  # every column with a valid key, padded query rows included, within the row maps' tolerance
            live = keep.any(1)  # [B, C]
            got = out["col_attentions"].cpu().permute(0, 3, 1, 2, 4, 5)  # [B, C, L, H, R, R]
            assert bool((got[~live] == 0).all()), "a column of padding only is not 0"
            ca = float((got.double() - ref["col_attentions"].permute(0, 3, 1, 2, 4, 5)).abs()[live].max())
        report(f"msa ragged batch precision={precision} need_head_weights={need}", repr_rel_fro=r, logits_rel_fro=lr,
               row_maps_max_abs=ra, col_maps_max_abs=ca)
        assert r <= tol[0] and lr <= tol[1] and ra <= tol[2] and ca <= tol[2]
    assert torch.equal(outs[0]["logits"], outs[1]["logits"])  # the maps change no bit of the rest
    assert torch.equal(outs[0]["representations"][L], outs[1]["representations"][L])
