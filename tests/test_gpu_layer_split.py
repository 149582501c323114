"""GPU (-m gpu): whole fp32x3 layers, for the parts of the split path only a layer reaches.

  * Narrow heads: one ESM-2 TransformerLayer with precision 1 at the 8M (d = 16), 150M (d = 32) and 650M (d = 64)
    widths against oracle.esm2_oracle.transformer_layer in float64 on the same fp32 parameters.  Heads narrower than 64
    sit in zero-padded 64-wide slots, so this is where the split pack_head_rows / pack_head_cols (lo halves at pitch 2E
    and 2Ea, Ea != E) run.
  * zero_q_at_pads_kernel<true>: the MSA axial stack is invariant to the values at padded positions.  The tied row
    attention sums q.k over the alignment rows with q zeroed at padded positions, and masks padded key columns, so
    nothing reaches a valid position from a padded one, bit for bit; in fp32x3 that needs q_lo zeroed as well."""
import pytest
import torch

from kernel_refs import layer64

pytestmark = pytest.mark.gpu

# Gates of the narrow-head layer test (DESIGN.md section 4 gives the measured maxima).  A lo weight half dropped or
# misplaced costs ~2^-12 = 2.4e-4 of its GEMM's output.
# Measured 6.3e-6 / 1.1e-5 / 2.2e-5 and 8.0e-6 / 1.6e-5 / 3.5e-5 at d = 16 / 32 / 64; the out_proj lo half written at
# the unslotted column moves the update by 1.5e-4 at d = 16 and 1.7e-4 at d = 32.
LAYER_DELTA_RELFRO = 4e-5   # rel-Frobenius of the layer's residual update (out - x) at the valid positions
LAYER_PROBS_MAX_ABS = 7e-5  # attention probabilities, valid query rows


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


@pytest.mark.parametrize("E,H", [(320, 20), (640, 20), (1280, 20)], ids=["8M", "150M", "650M"])
def test_narrow_head_layer_fp32x3_against_float64(E, H):
    from esm_b200.model import TransformerLayer
    from oracle.weights import make_state_dict
    T, B = 130, 2
    lengths = [130, 97]
    sd = make_state_dict(1, E, H, seed=E)
    layer = TransformerLayer(E, 4 * E, H)
    layer.load_state_dict({k[len("layers.0."):]: v for k, v in sd.items() if k.startswith("layers.0.")}, strict=True)
    layer = layer.cuda()
    layer.precision = 1
    x = torch.randn(T, B, E, generator=torch.Generator().manual_seed(E))
    pad = torch.zeros(B, T, dtype=torch.bool)
    for b, n in enumerate(lengths):
        pad[b, n:] = True
    with torch.no_grad():
        out, attn = layer(x.cuda(), self_attn_padding_mask=pad.cuda(), need_head_weights=True)  # (T,B,E), (H,B,T,T)
    torch.cuda.synchronize()
    sd64 = {k: v.double() for k, v in sd.items()}
    xb = x.transpose(0, 1).double()
    ref, p = layer64(xb, sd64, "layers.0.", H, pad)  # [B,T,E], [B,H,T,T]
    keep = ~pad
    got = out.transpose(0, 1).double().cpu()
    d_got, d_ref = (got - xb)[keep], (ref - xb)[keep]
    r = float((d_got - d_ref).norm() / d_ref.norm())
    pa = float((attn.transpose(0, 1).double().cpu() - p).abs()[keep[:, None, :, None].expand_as(p)].max())
    report(f"layer_split narrow heads E={E} H={H} d={E // H} T={T}", delta_rel_fro=r, probs_max_abs=pa)
    assert r <= LAYER_DELTA_RELFRO and pa <= LAYER_PROBS_MAX_ABS


@pytest.mark.parametrize("precision", [0, 1], ids=["fp16", "fp32x3"])
def test_axial_stack_is_invariant_to_padded_values(precision):
    """Two esmb200_axial_stack_forward calls on an MSA with trailing padded rows and columns, differing only in x at the
    padded positions: the outputs at valid positions and the row-attention entries between valid columns are
    bit-identical."""
    from esm_b200.msa import AxialTransformerLayer, run_axial_stack
    from oracle.msa_oracle import make_axial_state_dict
    E, Fd, H = 128, 512, 2
    B, R, C = 1, 9, 70
    sd = make_axial_state_dict(E, Fd, seed=3)
    layer = AxialTransformerLayer(E, Fd, H)
    layer.load_state_dict({k[len("layers.0."):]: v for k, v in sd.items()}, strict=True)
    layer = layer.eval().cuda()
    layer.precision = precision
    pad = torch.zeros(B, R, C, dtype=torch.bool, device="cuda")
    pad[:, R - 3:] = True     # trailing rows
    pad[:, :, C - 6:] = True  # trailing columns
    g = torch.Generator(device="cuda").manual_seed(11)
    x1 = torch.randn(B, R, C, E, device="cuda", generator=g)
    x2 = torch.where(pad[..., None], 3.0 * torch.randn(B, R, C, E, device="cuda", generator=g), x1)
    assert not torch.equal(x1, x2)
    y1, y2 = x1.clone(), x2.clone()
    a1 = run_axial_stack([layer], y1, pad, row_attn_layers=[0])[0]  # [H,B,C,C]
    a2 = run_axial_stack([layer], y2, pad, row_attn_layers=[0])[0]
    torch.cuda.synchronize()
    keep = ~pad
    cols = ~pad[:, 0]  # [B, C] valid columns
    both = cols[:, :, None] & cols[:, None, :]
    assert torch.equal(y1[keep], y2[keep])
    assert torch.equal(a1[:, both], a2[:, both])
    assert not torch.equal(y1, y2)  # the padded positions did differ
    report(f"layer_split pad invariance precision={precision} B={B} R={R} C={C}", valid_max_abs_diff=0.0,
           padded_max_abs_diff=float((y1 - y2).abs().max()))
