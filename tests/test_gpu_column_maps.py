"""GPU (-m gpu): the MSA Transformer's column attention maps at kernel precision, and column maps past the probability
kernel's 65535-index grid.

attention_probs_kernel writes the column maps of esmb200_axial_stack_forward ([B*C, H, R, R], ProbsParams::cols) from
the row statistics of the column attention's forward kernel.  One axial layer at E = 128, H = 2, F = 512 runs through
run_axial_stack with its column maps, in fp16 and fp32x3, and is replayed kernel by kernel (stack_replay.replay_axial):
the final x and the row maps must be the replay's bits, and the column maps are held to float64 on the replay's own
column q, k (stack_replay.attention_stage_f16 / attention_stage_split) at every query row of every column with a valid
key.  The column attention masks keys only and keeps q at padded rows (axial_attention.py:211-217), so the padded
query rows of a live column are softmax rows over the valid keys like any other.  Exact: padded keys 0, columns of
padding only 0 (the reference gives 1/R there: the documented deviation of msa.py), every map written (the buffer
starts as NaN).

Depths R around the 32-key words of the key bits, the 64- and 128-key blocks of the forward kernels, the 128-key tiles
of the probability kernel and its second query tile, up to 1024; widths C = 1, 3, 64, 65, 130; B = 1 and 2; no padding,
trailing padded columns, trailing padded rows of the last alignment (at R = 200 with depth 100 the second 128-key tile
of those columns is dead), and the ragged widths and depths of test_gpu_msa_key_padding.

R = 1 (the reference's all-ones special case, axial_attention.py:189): every live map is exactly 1.0, and in fp16 the
column ctx is v bit for bit.  The kernels do not special-case it.  The one weight is e = ex2.approx(fma(s, log2e,
-fp32(m log2e))) with m = s, the ex2 of the fp32 rounding residual of s log2e, so e = 1 + O(2^-13) rather than 1; the
probability is e * fp32(1 / l) with l = e, and e * fp32(1 / e) rounds to exactly 1 in fp32 for every |e - 1| < 2^-12.5
(all such fp32 values checked); in fp16 P = fp16(e) = 1 and ctx = fp16(v * fp32(1 / e)) = v.  In fp32x3, P lo = e - 1
is not 0: O = v hi + v lo + (e - 1) v hi, times fp32(1 / e), then split into hi | lo again, so ctx hi + lo is v hi + lo
only up to those fp32 roundings.  It is held to the float64 bound like every other case, and the deviation is
printed.

Past the grid: the probability kernel takes one grid z index per (sequence, head), so the library launches it once per
65535 / H sequences.  Checked at B*C = 32768, H = 2 (the second launch holds one sequence), at MSA-1b width with 6
alignments of 4 x 1024 tokens through the whole model, and for ESM-2 need_head_weights and fp32x3 predict_contacts at
B*H = 65540."""
import argparse

import pytest
import torch

import stack_replay as sr
from test_gpu_msa_key_padding import batch_mask

pytestmark = pytest.mark.gpu

E, FD, H = 128, 512, 2


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


_LAYERS = {}


def layer_for(precision):
    from esm_b200.msa import AxialTransformerLayer
    from oracle.msa_oracle import make_axial_state_dict
    if precision not in _LAYERS:
        sd = make_axial_state_dict(E, FD, seed=31)
        layer = AxialTransformerLayer(E, FD, H)
        layer.load_state_dict({k[len("layers.0."):]: v for k, v in sd.items()}, strict=True)
        layer = layer.eval().cuda()
        layer.precision = precision
        _LAYERS[precision] = (layer, sr.pack_axial(layer, precision))
    return _LAYERS[precision]


def make_pad(kind, B, R, C):
    """[B,R,C] bool on the device, or None"""
    if kind == "none":
        return None
    pad = torch.zeros(B, R, C, dtype=torch.bool)
    if kind == "cols":  # trailing fully padded columns
        pad[:, :, C - max(1, C // 5):] = True
    elif kind == "rows":  # trailing padded rows of the last alignment, and one padded column
        pad[B - 1, (R + 1) // 2:] = True
        pad[:, :, C - 1] = True
    elif kind == "ragged":  # alignment b: depths[b] rows of widths[b] columns (MSABatchConverter's padding)
        widths = [C, (3 * C) // 4, max(1, C // 6)][:B]
        depths = [R, max(1, (2 * R) // 3), max(1, R // 2)][:B]
        pad = batch_mask(widths, depths, R, C)
    return pad.cuda()


def run_and_replay(precision, B, R, C, pad, seed):
    """the layer through run_axial_stack with row and column maps, and through the replay; returns (column maps
    [B,C,H,R,R], replay stages, cpad [B*C,R])"""
    from esm_b200.msa import run_axial_stack
    layer, pk = layer_for(precision)
    M = B * R * C
    x0 = torch.randn(B, R, C, E, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed))
    xa, xr = x0.clone(), x0.clone()
    col = torch.full((B, C, H, R, R), float("nan"), device="cuda")
    ra = run_axial_stack([layer], xa, pad, row_attn_layers=[0], col_attn={0: col})[0]
    rr = torch.empty(H, B, C, C, device="cuda")
    st = sr.replay_axial(layer, pk, xr.view(M, E), pad, B, R, C, precision, rr)
    torch.cuda.synchronize()
    assert torch.equal(xa, xr), "run_axial_stack and the replay differ"
    assert torch.equal(ra, rr), "row attention maps differ from the replay's"
    assert not bool(col.isnan().any()), "a column map was not written"
    cpad = (pad.permute(0, 2, 1).reshape(B * C, R) if pad is not None else
            torch.zeros(B * C, R, dtype=torch.bool, device="cuda"))
    return col, st, cpad


def check_column_maps(precision, col, st, cpad, B, R, C):
    """the column maps and ctx against float64 on the replay's column q, k, v; exact zeros; worst ratios"""
    N = B * C
    cp = col.view(N, H, R, R)
    sr.column_zero_stage("column maps", cp, cpad)
    cq, cc = sr._column_major(st["col_qkv"], B, R, C), sr._column_major(st["col_ctx"], B, R, C)
    qrows = sr.column_query_rows(cpad)
    worst = {}
    if precision:
        sr.attention_stage_split(worst, cq, cc, cpad, N, R, H, cp, prefix="col_", qrows=qrows)
    else:
        sr.attention_stage_f16(worst, cq, cc, cpad, N, R, H, cp, blocks=(64, 128), prefix="col_", qrows=qrows)
    return worst


# (B, R, C, padding): every R of the sweep, B*C*H*R^2 at most about 10^7
CASES = [
    (2, 1, 130, "cols"), (1, 1, 1, "none"), (2, 2, 65, "rows"), (1, 31, 64, "none"), (2, 32, 65, "cols"),
    (2, 33, 3, "rows"), (1, 63, 130, "none"), (2, 64, 64, "rows"), (1, 65, 65, "cols"), (2, 127, 3, "none"),
    (1, 128, 64, "cols"), (2, 128, 3, "rows"), (2, 129, 65, "cols"), (2, 200, 64, "rows"), (1, 1000, 3, "cols"),
    (2, 1024, 3, "rows"), (3, 6, 70, "ragged"), (3, 130, 64, "ragged"),
]


@pytest.mark.parametrize("precision", [0, 1], ids=["fp16", "fp32x3"])
@pytest.mark.parametrize("B,R,C,kind", CASES, ids=[f"{b}x{r}x{c}-{k}" for b, r, c, k in CASES])
def test_column_maps_against_float64(B, R, C, kind, precision):
    pad = make_pad(kind, B, R, C)
    col, st, cpad = run_and_replay(precision, B, R, C, pad, seed=R * 1000 + C)
    worst = check_column_maps(precision, col, st, cpad, B, R, C)
    label = f"column maps {B}x{R}x{C} {kind} p{precision}"
    for name, r in worst.items():
        report(f"{label} {name}", worst=r)
    for name, r in worst.items():
        assert r <= 1.0, (label, name, r)
    if R == 1:
        live = ~cpad[:, 0]  # [B*C]: a column of one token is live when that token is not padding
        assert bool((col.view(B * C, H)[live] == 1.0).all()), "a one-key column map is not exactly 1"
        v = sr._column_major(st["col_qkv"], B, R, C)
        ctx = sr._column_major(st["col_ctx"], B, R, C)
        if precision:  # within the float64 bound above, not bit for bit (module docstring); the deviation is printed
            vs = v[live, 2 * E:3 * E].double() + v[live, 5 * E:].double()
            cs = ctx[live, :E].double() + ctx[live, E:].double()
            report(f"{label} ctx hi + lo vs v hi + lo at R = 1", max_rel=float(((cs - vs).abs() / vs.abs()).max()),
                   differing=float((cs != vs).sum()), of=float(cs.numel()))
        else:
            assert torch.equal(ctx[live], v[live, 2 * E:3 * E]), "fp16: ctx is not v at R = 1"


# ---- past the probability kernel's grid -----------------------------------------------------------------------------
def test_column_maps_of_32768_sequences_in_two_launches():
    """B*C = 32768 column sequences at H = 2: 65536 maps, one past the grid; the second launch holds exactly one
    sequence (the last column of the last alignment).  Against float64, and the same bits as the two halves run
    alone."""
    from esm_b200.msa import run_axial_stack
    precision, B, R, C = 0, 32, 2, 1024
    pad = torch.zeros(B, R, C, dtype=torch.bool, device="cuda")
    pad[B - 1, 1:, C - 300:] = True  # the last sequence has one valid key and a padded query row
    col, st, cpad = run_and_replay(precision, B, R, C, pad, seed=77)
    worst = check_column_maps(precision, col, st, cpad, B, R, C)
    for name, r in worst.items():
        report(f"column maps {B}x{R}x{C} two launches p{precision} {name}", worst=r)
    for name, r in worst.items():
        assert r <= 1.0, (name, r)
    layer, _ = layer_for(precision)
    x0 = torch.randn(B, R, C, E, device="cuda", generator=torch.Generator(device="cuda").manual_seed(77))
    for lo, hi in ((0, B // 2), (B // 2, B)):
        xh = x0[lo:hi].clone()
        ch = torch.full((hi - lo, C, H, R, R), float("nan"), device="cuda")
        run_axial_stack([layer], xh, pad[lo:hi].contiguous(), col_attn={0: ch})
        torch.cuda.synchronize()
        assert torch.equal(ch, col[lo:hi]), f"alignments {lo}..{hi - 1}: maps differ from the batched call"


def msa_model(L, E_, F_, H_, seed):
    from esm_b200.msa import MSATransformer
    from oracle import msa_oracle
    sd = msa_oracle.make_msa_state_dict(L, E_, F_, H_, seed=seed)
    model = MSATransformer(argparse.Namespace(layers=L, embed_dim=E_, ffn_embed_dim=F_, attention_heads=H_,
                                              max_positions=1024, embed_positions_msa=True))
    model.load_state_dict(sd, strict=True)
    return model.eval().cuda()


def test_msa1b_width_six_alignments_of_1024_columns_with_contacts():
    """6 alignments of 4 x 1024 tokens at MSA-1b width (H = 12): 73,728 column maps per layer.  model(tokens,
    return_contacts=True) runs, and each alignment's logits, row maps, column maps and contacts are the bits of that
    alignment run alone."""
    from oracle import msa_oracle
    model = msa_model(2, 768, 3072, 12, seed=6)
    tokens = msa_oracle.make_msa_tokens(6, 4, 1024, seed=13).cuda()
    out = model(tokens, return_contacts=True)
    torch.cuda.synchronize()
    assert out["col_attentions"].shape == (6, 2, 12, 1024, 4, 4)
    bad = {}
    for b in range(6):
        one = model(tokens[b:b + 1], return_contacts=True)
        for key in ("logits", "row_attentions", "col_attentions", "contacts"):
            bad[key] = bad.get(key, 0) + int((one[key][0] != out[key][b]).sum())
    report("msa1b 6x4x1024 return_contacts alone vs batched", **{k: float(v) for k, v in bad.items()})
    assert all(v == 0 for v in bad.values()), bad


@pytest.mark.parametrize("precision", ["fp16", "fp32x3"])
def test_esm2_maps_past_the_grid(precision):
    """ESM-2 at 8M width (E 320, H 20) with B = 65535 // 20 + 1 = 3277 short sequences: fp16 need_head_weights maps,
    and fp32x3 predict_contacts (its maps go through the split probability kernel), equal the same sequences run in two
    batches below the limit, bit for bit."""
    from esm_b200 import ESM2
    from oracle.weights import make_state_dict, make_tokens
    L, E_, H_ = 2, 320, 20
    B = 65535 // H_ + 1
    model = ESM2(num_layers=L, embed_dim=E_, attention_heads=H_)
    model.load_state_dict(make_state_dict(L, E_, H_, seed=2), strict=True)
    model = model.eval().cuda().set_precision(precision)
    g = torch.Generator().manual_seed(3)
    tokens = make_tokens(torch.randint(1, 11, (B,), generator=g).tolist(), 12, seed=4).cuda()
    halves = ((0, B // 2), (B // 2, B))
    if precision == "fp16":
        got = model(tokens, need_head_weights=True)["attentions"]
        parts = [model(tokens[lo:hi], need_head_weights=True)["attentions"] for lo, hi in halves]
    else:
        got = model.predict_contacts(tokens)
        parts = [model.predict_contacts(tokens[lo:hi]) for lo, hi in halves]
    torch.cuda.synchronize()
    bad = int((torch.cat(parts) != got).sum())
    report(f"esm2 8M width B={B} {precision} past the grid vs two batches", mismatches=float(bad),
           max_abs=float(got.abs().max()))
    assert bad == 0
