"""CPU: the float64 references of tests/kernel_refs.py that the kernel-level GPU tests compare against.

  * the contact partials, summed, give the reference contact head (oracle.esm2_oracle.contact_head) on random maps, and
    each partial is the sum over its own 32-wide quarter (a swapped quarter or tile index in the reference fails here);
  * the per-model GEMM launch table reproduces the packed layer size the library reports and the shapes of the models'
    own modules;
  * the erf-GELU bound holds for an fp32 restatement of the epilogue's formula;
  * the fp16 attention bounds hold for a float64 emulation of the kernels' arithmetic, are not vacuous, and refuse the
    same emulation with a padded key counted, a block's O rescale skipped or ctx scaled by 1 + 2^-9; the reference
    over slices of query rows equals the whole-head reference bit for bit; the bounds hold with up to 64 key blocks
    (T = 4096 and 8192) and refuse the O rescale skipped from the 9th block on;
  * the tied row attention's stage and end-to-end bounds hold for a float64 emulation of its three kernels in fp16 and
    fp32x3, and refuse P x (1 + 2^-13), ctx x (1 + 2^-9), an alignment row's slab dropped from the logits, the split
    slab's q_lo k_hi pass dropped, and V read from the next alignment row;
  * the embedding references give the oracles' embeddings (oracle.esm2_oracle.embed, the embedding lines of
    oracle.msa_oracle.msa_transformer_forward, its representation 0), positions a hand-written example, mean_pool64 and
    log_softmax64 torch's float64 results, contact_stripes the reference contact head, and layer64 the oracle's layer;
    torch's fp32 log-softmax stays inside log_softmax_bound and a row summed over its first 32 columns only does not;
  * heads in 64-wide slots at widths 8 .. 128: the replay's slot map is elementwise.cuh's head_slot and inverts; the
    kernel's (c, c + 32) rotation on the packed heads is the reference's rotate-half; qkv_ref_heads is qkv_ref at
    d = 64; an fp32 restatement of the QKV epilogue stays inside qkv_bound, and a neighbouring table column or a pair in
    the head's other slot leaves it."""
import math

import numpy as np
import pytest
import torch

import kernel_refs as kr


def _random_maps(L, B, H, T, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.rand(B, L, H, T, T, generator=g, dtype=torch.float64)
    return a / a.sum(-1, keepdim=True)


@pytest.mark.parametrize("T,lengths", [(40, [38, 20]), (129, [127, 60]), (300, [298, 100])])
def test_contact_partials_sum_to_the_reference_contact_head(T, lengths):
    from oracle import esm2_oracle
    from oracle.weights import make_tokens
    L, H = 2, 3
    tokens = make_tokens(lengths, T, seed=T)
    B = len(lengths)
    attn = _random_maps(L, B, H, T, seed=T + 1)
    g = torch.Generator().manual_seed(T + 2)
    sd = {"contact_head.regression.weight": torch.randn(1, L * H, generator=g, dtype=torch.float64),
          "contact_head.regression.bias": torch.randn(1, generator=g, dtype=torch.float64)}
    want = esm2_oracle.contact_head(tokens, attn, sd)
    keep = tokens.ne(2)
    w = sd["contact_head.regression.weight"].view(L, H)
    parts = [kr.contact_partials(attn[:, l], w[l], keep, 1, T - 1) for l in range(L)]
    acc = sum(p[0] for p in parts)
    row = torch.stack([p[1] for p in parts])
    col = torch.stack([p[2] for p in parts])
    nt = (T + 127) // 128
    assert row.shape == col.shape == (L, B, H, 4 * nt, T - 2)
    got = kr.contacts_from_partials(acc, row, col, w, float(sd["contact_head.regression.bias"]))
    torch.testing.assert_close(got, want, atol=1e-12, rtol=1e-12)


def test_contact_partials_are_per_quarter():
    """Each partial is the sum over exactly its 32 keys (rows) / 32 queries (columns) of the cropped, masked maps."""
    T, lo, hi = 300, 1, 299
    attn = _random_maps(1, 2, 2, T, seed=5)[:, 0]
    keep = torch.ones(2, T, dtype=torch.bool)
    keep[1, 150] = False
    _, row, col = kr.contact_partials(attn, torch.ones(2), keep, lo, hi)
    a = kr.masked_maps(attn, keep, lo, hi)
    for p in range(row.shape[2]):
        kt, q = divmod(p, 4)
        j0 = 128 * kt + 32 * q
        torch.testing.assert_close(row[:, :, p], a[:, :, lo:hi, j0:j0 + 32].sum(-1), atol=0, rtol=1e-14)
        torch.testing.assert_close(col[:, :, p], a[:, :, j0:j0 + 32, lo:hi].sum(-2), atol=0, rtol=1e-14)
    assert float(row[:, :, 10:].abs().max()) == 0.0  # quarters that start at or past T = 300 (320, 352, ...) are empty
    assert float(row[0, :, 9].abs().min()) > 0.0     # quarter 9 holds keys 288 .. 298
    assert float(row[1, :, :, 150 - lo].abs().max()) == 0.0 and float(col[1, :, :, 150 - lo].abs().max()) == 0.0


@pytest.mark.parametrize("name", sorted(kr.MODELS))
def test_gemm_launch_table_matches_the_packed_layer(name):
    from esm_b200 import _lib
    _, E, H, F, _, msa = kr.MODELS[name]
    if msa:  # the MSA layer's feed-forward half is packed by the column layer: check the attention GEMMs instead
        launches = kr.gemm_launches(name)
        assert [(e, n, k) for _, e, n, k in launches[:4]] == [(kr.EPI_QKV_ROPE, 3 * E, E),
                                                            (kr.EPI_BIAS_RESIDUAL, E, E)] * 2
    else:
        assert _lib.load().esmb200_layer_packed_bytes(E, H, F, 0) == kr.packed_bytes_from_launches(name)


@pytest.mark.parametrize("name", ["esm2_t6_8M", "esm2_t12_35M", "esm1b_t33_650M", "esm_msa1b_t12_100M"])
def test_gemm_launch_table_matches_the_modules(name):
    """The K and N of the table are the in/out features of the modules the model builds (unpadded for head_dim 64
    and below; the LM head's projection padded to 64 vocabulary rows)."""
    n_layers, E, H, F, rotary, msa = kr.MODELS[name]
    launches = {role: (n, k) for role, _, n, k in kr.gemm_launches(name)}
    if msa:
        from argparse import Namespace
        from esm_b200.msa import MSATransformer
        m = MSATransformer(Namespace(layers=1, embed_dim=E, ffn_embed_dim=F, attention_heads=H, max_positions=1024,
                                     embed_positions_msa=True))
        layer = m.layers[0]
        ffn = layer.feed_forward_layer.layer
        assert launches["out_proj"] == tuple(layer.row_self_attention.layer.out_proj.weight.shape)
    else:
        from esm_b200 import ESM2
        from esm_b200.model import TransformerLayer
        layer = TransformerLayer(E, F, H, rotary)
        ffn = layer
        # heads narrower than 64 sit in zero-padded 64-wide slots: q, k and v are 64 * H wide on the attention side
        Ea = 64 * kr.head_slots(E, H) * H
        assert Ea >= layer.self_attn.q_proj.out_features and (Ea == E) == (E // H == 64)
        assert launches["qkv"] == (3 * Ea, layer.self_attn.q_proj.in_features)
        assert launches["out_proj"] == (layer.self_attn.out_proj.out_features, Ea)
        if name.startswith("esm2"):
            assert ESM2(num_layers=1, embed_dim=E, attention_heads=H).lm_head.weight.shape == (kr.VOCAB, E)
    assert launches["fc1"] == tuple(ffn.fc1.weight.shape) and launches["fc2"] == tuple(ffn.fc2.weight.shape)
    assert launches["lm_dense"] == (E, E) and launches["lm_out"] == (64, E)


def test_split16_is_exact_hi_plus_rounded_residue():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(10000, generator=g) * torch.logspace(-8, 4, 10000)  # below the fp16 overflow at 65520
    hi, lo = kr.split16(x)
    assert hi.dtype == lo.dtype == torch.float16
    assert torch.equal(hi, x.half())
    assert torch.equal(lo, (x.double() - hi.double()).float().half())  # x - hi is exact in fp32
    assert torch.equal(kr.join64(hi, lo), hi.double() + lo.double())


def test_split_representation_bound_holds_and_is_tight():
    """|x - (hi + lo)| <= 2^-22 |x| + 2^-25 from 1e-8 to 6e4, and the bound is attained to within 2x: overall (lo
    subnormal) and on the normal range alone (where the largest error is half the 2^-22 term)."""
    g = torch.Generator().manual_seed(1)
    mag = torch.logspace(-8, math.log10(6e4), 400001, dtype=torch.float64)
    x = (mag * torch.where(torch.rand(mag.shape, generator=g) < 0.5, -1.0, 1.0)).float()
    hi, lo = kr.split16(x)
    assert bool(torch.isfinite(hi).all())
    err = (x.double() - kr.join64(hi, lo)).abs()
    ratio = err / kr.split_rep_bound(x)
    assert float(ratio.max()) <= 1.0
    assert float(ratio.max()) >= 0.5
    big = x.abs() >= 1.0
    assert float(ratio[big].max()) >= 0.45
    assert float(ratio[x.abs() < 2.0 ** -3].max()) >= 0.5  # the subnormal half-quantum is needed
    assert float((err / (2.0 ** -22 * x.double().abs()))[x.abs() < 2.0 ** -3].max()) > 1.0


def test_fp32x3_models_follow_set_precision():
    """kr.FP32X3_MODELS are exactly the table's models whose set_precision("fp32x3") succeeds (the MSA layers have
    head_dim 64 by construction)"""
    from types import SimpleNamespace
    from esm_b200.model import ProteinLanguageModel
    assert kr.FP32X3_MODELS == ["esm2_t6_8M", "esm2_t30_150M", "esm2_t33_650M", "esm2_t36_3B", "esm1b_t33_650M",
                                "esm_msa1b_t12_100M"]
    for name, (_, E, H, _, _, msa) in kr.MODELS.items():
        if msa:
            assert E == 64 * H and name in kr.FP32X3_MODELS
            continue
        stub = SimpleNamespace(embed_dim=E, attention_heads=H, PRECISIONS=ProteinLanguageModel.PRECISIONS,
                               precision="fp16", layers=[SimpleNamespace(precision=0)], _offload=None)
        try:
            ProteinLanguageModel.set_precision(stub, "fp32x3")
            ok = True
        except ValueError:
            ok = False
        assert ok == (name in kr.FP32X3_MODELS), name
        assert not ok or stub.layers[0].precision == 1


def test_split_acc_bound_covers_an_emulated_three_pass_product():
    """The three-pass product with fp32 accumulation in k16 steps truncated toward zero (the tensor core's behaviour,
    emulated in float64 then chopped to fp32) stays inside kr.split_acc_bound, and dropping a pass does not."""
    g = torch.Generator().manual_seed(2)
    M, N, K = 16, 24, 640
    a, w = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) * K ** -0.5
    ah, al = kr.split16(a)
    wh, wl = kr.split16(w)
    y = kr.join64(ah, al) @ kr.join64(wh, wl).t()

    def chop(t):  # round toward zero to fp32
        f = t.float()
        over = f.double().abs() > t.abs()
        return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f).double()

    def run(passes):
        acc = torch.zeros(M, N, dtype=torch.float64)
        for k0 in range(0, K, 64):
            for pa, pw in passes:
                for s in range(k0, k0 + 64, 16):
                    acc = chop(acc + pa[:, s:s + 16].double() @ pw[:, s:s + 16].double().t())
        return acc

    b = kr.split_acc_bound(ah, al, wh, wl, K, y)
    good = run([(ah, wh), (al, wh), (ah, wl)])
    assert float(((good - y).abs() / b).max()) <= 1.0
    bad = run([(ah, wh), (ah, wh), (ah, wl)])  # lo*hi read as hi*hi
    assert float(((bad - y).abs() / b).max()) > 1.0
    dropped = run([(ah, wh), (ah, wl)])        # lo*hi missing
    assert float(((dropped - y).abs() / b).max()) > 1.0


def test_gelu_bound_covers_an_fp32_restatement():
    """The epilogue's formula evaluated in fp32 with correctly rounded reciprocal and exponential stays inside the bound
    (the approximate MUFU instructions' share of the bound is not exercised here; the GPU test does that)."""
    assert kr.horner_condition() <= 4.0
    x = np.concatenate([np.linspace(-12, 12, 200001), np.linspace(-1e-3, 1e-3, 20001)]).astype(np.float32)
    f = np.float32
    z = np.abs(x) * f(0.70710678118654752440)
    t = f(1) / (f(0.3275911) * z + f(1))
    poly = f(0.5 * 1.061405429) * t + f(0.5 * -1.453152027)
    for c in (0.5 * 1.421413741, 0.5 * -0.284496736, 0.5 * 0.254829592):
        poly = poly * t + f(c)
    poly = poly * t
    e = np.exp2(z * (z * f(-1.4426950408889634))).astype(np.float32)
    q = poly * e
    y = x * np.where(x >= 0, f(1) - q, q)
    xt = torch.from_numpy(x.astype(np.float64))
    err = (torch.from_numpy(y.astype(np.float64)) - kr.gelu64(xt)).abs()
    bound = kr.gelu_bound(xt)
    assert bool((err <= bound).all()), float((err / bound).max())
    assert float((err / bound).max()) > 0.05  # the bound is not vacuous
    assert math.isclose(float(kr.gelu64(torch.tensor(1.0))), 0.8413447460685429, rel_tol=1e-15)


# ---- fp16 attention -------------------------------------------------------------------------------------------------
LOG2E32 = float(torch.tensor(1.4426950408889634, dtype=torch.float32))


def _f32(t):
    return t.float().double()


def _chop(t):  # round toward zero to fp32: the tensor core's accumulation
    f = t.float()
    over = f.double().abs() > t.abs()
    return torch.where(over, torch.nextafter(f, torch.zeros_like(f)), f).double()


def _emulate_attention(q, k, v, padded, block, count_key=None, skip_rescale=None, skip_rescale_from=None):
    """float64 emulation of the fp16 attention kernels' arithmetic on one head: q [Tq, D] (any Tq of the head's query
    rows), k, v [T, D] fp16, padded [T] bool.  Logits in fp32 truncating k16 steps; per `block`-key block the exact
    running maximum, e = 2^(fp32(s log2e - m log2e)) (correctly rounded: ex2.approx's own error is not emulated),
    l = fp32(alpha l + fp32 sum e), P = fp16(e), O = fp32(alpha O) + P V in truncating k16 steps;
    ctx = fp16(O * fp32(1 / l)).  Returns ctx, the saved row max and row sum, and the probability kernel's output from
    the same logits.  Faults: count_key (a padded key index counted as attendable), skip_rescale (a block index whose O
    rescale is left out), skip_rescale_from (the O rescale left out from this block index on)."""
    Tq, D = q.shape
    T = k.shape[0]
    live = ~padded
    if count_key is not None:
        live = live.clone()
        live[count_key] = True
    kvlen = int(torch.nonzero(live).max()) + 1 if bool(live.any()) else 0
    s = torch.zeros(Tq, T, dtype=torch.float64)
    for d0 in range(0, D, 16):
        s = _chop(s + q[:, d0:d0 + 16].double() @ k[:, d0:d0 + 16].double().t())
    s = s.masked_fill(~live[None, :], float("-inf"))
    m = torch.full((Tq, 1), float("-inf"), dtype=torch.float64)
    l = torch.zeros(Tq, 1, dtype=torch.float64)
    o = torch.zeros(Tq, D, dtype=torch.float64)
    for j0 in range(0, kvlen, block):
        sb = s[:, j0:j0 + block]
        mn = torch.maximum(m, sb.amax(-1, keepdim=True))
        alpha = torch.where(torch.isinf(mn), torch.ones_like(mn), torch.exp2(_f32(_f32(m - mn) * LOG2E32)))
        ref = torch.where(torch.isinf(mn), torch.zeros_like(mn), _f32(-mn * LOG2E32))
        e = _f32(torch.exp2(_f32(sb * LOG2E32 + ref)))
        m = mn
        l = _f32(_f32(l * alpha) + _f32(e.float().sum(-1, keepdim=True)))
        if j0 // block != skip_rescale and (skip_rescale_from is None or j0 // block < skip_rescale_from):
            o = _f32(o * alpha)
        ph = e.half().double()
        vb = v[j0:j0 + block].double()
        for k0 in range(0, ph.shape[1], 16):
            o = _chop(o + ph[:, k0:k0 + 16] @ vb[k0:k0 + 16])
    inv = torch.where(l > 0, _f32(1.0 / torch.where(l > 0, l, torch.ones_like(l))), torch.zeros_like(l))
    ctx = _f32(o * inv).half().double()
    mx = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    probs = _f32(_f32(torch.exp2(_f32(s * LOG2E32 + _f32(-mx * LOG2E32)))) * inv)
    return ctx, mx[:, 0], l[:, 0], probs


def _attention_inputs(T, D, std, seed, rise=False):
    """fp16 q, k, v [T, D] with logits of std `std` (diffuse at 1, sharp at 8); rise: every 64 keys score ~3 higher"""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(T, D, generator=g, dtype=torch.float64) * std / math.sqrt(D)
    k = torch.randn(T, D, generator=g, dtype=torch.float64)
    if rise:
        u = q.mean(0)
        k = k + (torch.arange(T, dtype=torch.float64) // 64)[:, None] * 3.0 * u / float(u @ u)
    v = torch.randn(T, D, generator=g, dtype=torch.float64)
    return q.half(), k.half(), v.half()


def _ratios(q, k, v, padded, block, ctx, mx=None, sm=None, probs=None):
    r = kr.attention64(q[None, None], k[None, None], v[None, None], padded[None], block)
    out = {"ctx": float(((ctx - r["ctx"][0, 0]).abs() / kr.attn_ctx_bound(r)[0, 0]).max())}
    num = (ctx - r["ctx"][0, 0]).pow(2).sum().sqrt()
    out["gate"] = float(num / r["ctx"].pow(2).sum().sqrt() / kr.attn_relfro_gate(r)[0, 0])
    if mx is not None:
        out["max"] = float(((mx - r["m"][0, 0, :, 0]).abs() / kr.attn_max_bound(r)[0, 0]).max())
        l_at = torch.exp(r["s"].masked_fill(r["km"], float("-inf")) - mx[None, None, :, None]).sum(-1)
        out["sum"] = float(((sm - l_at[0, 0]).abs() / kr.attn_sum_bound(r, l_at)[0, 0]).max())
        out["probs"] = float(((probs - r["p"][0, 0]).abs() / kr.attn_probs_bound(r)[0, 0]).max())
        live = ~padded.all()
        dev = (probs.sum(-1) - 1).abs() if bool(live) else torch.zeros(probs.shape[0], dtype=torch.float64)
        out["rowsum"] = float((dev / kr.attn_rowsum_bound(r)[0, 0]).max())
    return out


ATTN_EMU_CASES = [(300, 64, 128, 1.0, False), (300, 64, 128, 8.0, False), (1024, 64, 128, 1.0, False),
                  (300, 128, 64, 1.0, False), (300, 128, 64, 8.0, False), (400, 128, 64, 2.0, True),
                  (400, 64, 128, 2.0, True)]


@pytest.mark.parametrize("T,D,block,std,rise", ATTN_EMU_CASES)
def test_attention_bounds_cover_an_emulated_kernel(T, D, block, std, rise):
    """The emulated kernel, on a ragged mask with the last key padded, stays inside every bound; the bounds are not
    vacuous: the worst element of ctx reaches 0.1 of its bound and the gate 0.1 (diffuse heads, where neither term is
    dominated by exact one-hot rows)."""
    q, k, v = _attention_inputs(T, D, std, seed=T + D + int(std))
    padded = torch.zeros(T, dtype=torch.bool)
    padded[T - 37:] = True
    padded[5:9] = True
    ctx, mx, sm, probs = _emulate_attention(q, k, v, padded, block)
    out = _ratios(q, k, v, padded, block, ctx, mx, sm, probs)
    assert max(out.values()) <= 1.0, out
    if std == 1.0:
        assert out["ctx"] >= 0.1 and out["gate"] >= 0.1, out


@pytest.mark.parametrize("D,block", [(64, 128), (128, 64)])
def test_attention_bounds_refuse_emulated_faults(D, block):
    """The same emulation with one padded key counted, one block's O rescale skipped, or ctx scaled by 1 + 2^-9
    leaves the element bound or the per-head gate; probabilities scaled by 1 + 2^-13 leave the row-sum bound, which is
    tighter than the sum of the element bounds (that sum is implied by the element check and refuses nothing on its
    own)."""
    T = 300
    q, k, v = _attention_inputs(T, D, 2.0, seed=7, rise=True)
    padded = torch.zeros(T, dtype=torch.bool)
    padded[T - 37:] = True
    good, _, _, _ = _emulate_attention(q, k, v, padded, block)
    assert max(_ratios(q, k, v, padded, block, good).values()) <= 1.0
    counted, _, _, _ = _emulate_attention(q, k, v, padded, block, count_key=T - 20)
    skipped, _, _, _ = _emulate_attention(q, k, v, padded, block, skip_rescale=1)
    for bad in (counted, skipped):
        assert max(_ratios(q, k, v, padded, block, bad).values()) > 1.0
    qd, kd, vd = _attention_inputs(1024, D, 1.0, seed=8)
    pd = torch.zeros(1024, dtype=torch.bool)
    ctx, mx, sm, probs = _emulate_attention(qd, kd, vd, pd, block)
    scaled = (ctx * (1 + 2.0 ** -9)).half().double()
    assert _ratios(qd, kd, vd, pd, block, scaled)["gate"] > 1.0
    up = _f32(probs * (1 + 2.0 ** -13))
    assert _ratios(qd, kd, vd, pd, block, ctx, mx, sm, up)["rowsum"] > 1.0
    r = kr.attention64(qd[None, None], kd[None, None], vd[None, None], pd[None], block)
    dev = (up.sum(-1) - 1).abs()
    summed = float((dev / kr.attn_probs_bound(r)[0, 0].sum(-1)).max())
    assert float((dev / kr.attn_rowsum_bound(r)[0, 0]).max()) > 1.3 * summed  # tighter than the summed element bounds


# ---- long heads: row slices and up to 64 key blocks ------------------------------------------------------------------
def test_row_slices_equal_the_whole_head():
    """attention64_rows gives every row-indexed value and bound of attention64 on the whole head bit for bit (rows
    are independent), the same nblk, and the whole head's gate from the slices' summed terms; slices of 37 rows leave
    a short last one, and one sequence is all padding."""
    g = torch.Generator().manual_seed(11)
    B, H, T, D = 3, 2, 300, 64
    q, k, v = (torch.randn(B, H, T, D, generator=g).half() for _ in range(3))
    padded = torch.zeros(B, T, dtype=torch.bool)
    padded[1, 171:] = True
    padded[2] = True
    whole = kr.attention64(q, k, v, padded, 128)
    l_at = torch.exp(whole["s"].masked_fill(whole["km"], float("-inf")) - whole["m"]).sum(-1)
    bounds = {"ctx": kr.attn_ctx_bound(whole), "probs": kr.attn_probs_bound(whole),
              "rowsum": kr.attn_rowsum_bound(whole), "max": kr.attn_max_bound(whole),
              "sum": kr.attn_sum_bound(whole, l_at)}
    terms = [torch.zeros(B, H, dtype=torch.float64) for _ in range(3)]
    starts = []
    for i0, r in kr.attention64_rows(q, k, v, padded, 128, max_elems=B * H * T * 37):
        n = r["q"].shape[-2]
        starts.append((i0, n))
        rows = slice(i0, i0 + n)
        for name in ("s", "m", "l", "p", "ctx", "lerr", "delta"):
            assert torch.equal(r[name], whole[name][:, :, rows]), name
        assert torch.equal(r["nblk"], whole["nblk"])
        la = torch.exp(r["s"].masked_fill(r["km"], float("-inf")) - r["m"]).sum(-1)
        got = {"ctx": kr.attn_ctx_bound(r), "probs": kr.attn_probs_bound(r), "rowsum": kr.attn_rowsum_bound(r),
               "max": kr.attn_max_bound(r), "sum": kr.attn_sum_bound(r, la)}
        for name, b in got.items():
            assert torch.equal(b, bounds[name][:, :, rows]), name
        for acc, t in zip(terms, kr.attn_relfro_terms(r)):
            acc += t
    assert starts[0] == (0, 37) and starts[-1] == (296, 4) and len(starts) == 9
    torch.testing.assert_close(kr.attn_relfro_combine(*terms), kr.attn_relfro_gate(whole), rtol=1e-13, atol=0)
    assert [int(x) for x in whole["nblk"].flatten()] == [3, 2, 0]


def _rising_inputs(T, D, seed):
    """fp16 q, k, v [T, D] whose logits rise by ~3.2 every 64 keys (tests/test_gpu_attention_f16.py rising_qkv):
    every 64-key step of every row raises the running maximum, so every block rescales O and l"""
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(D, generator=g, dtype=torch.float64)
    u = u / u.norm() * 8.0 ** 0.5
    blk = (torch.arange(T, dtype=torch.float64) // 64)[:, None]
    q = u + 0.1 * torch.randn(T, D, generator=g, dtype=torch.float64)
    k = u * (0.4 * blk) + 0.3 * torch.randn(T, D, generator=g, dtype=torch.float64)
    v = torch.randn(T, D, generator=g, dtype=torch.float64)
    return q.half(), k.half(), v.half()


def _long_inputs(T, D, std, rise, seed):
    """(q rows, k, v, padded): 96 query rows spread over the head (rows are independent, so they stand for all T),
    keys padded at the tail and in one interior run"""
    q, k, v = _rising_inputs(T, D, seed) if rise else _attention_inputs(T, D, std, seed)
    padded = torch.zeros(T, dtype=torch.bool)
    padded[T - 37:] = True
    padded[T // 3:T // 3 + 5] = True
    return q[torch.arange(0, T, T // 96)], k, v, padded


LONG_EMU_CASES = [(64, 128, 8192, 1.0, False), (64, 128, 8192, 8.0, False), (64, 128, 4096, 2.0, True),
                  (128, 64, 4096, 1.0, False), (128, 64, 4096, 8.0, False), (128, 64, 4096, 2.0, True)]


@pytest.mark.parametrize("D,block,T,std,rise", LONG_EMU_CASES)
def test_attention_bounds_cover_an_emulated_kernel_to_64_blocks(D, block, T, std, rise):
    """nblk up to 64 (the wg kernel at T = 8192, the two-slot kernel at 4096): the bounds' nblk terms still cover the
    emulated kernel.  They are worst cases linear in nblk, so the worst ratio of a diffuse head falls with T (0.05 for
    ctx and the gate at 64 blocks of 128 keys, against 0.1 .. 0.3 at T <= 1024); 0.03 keeps them from going vacuous."""
    q, k, v, padded = _long_inputs(T, D, std, rise, seed=T + D + int(std))
    ctx, mx, sm, probs = _emulate_attention(q, k, v, padded, block)
    r = kr.attention64(q[None, None], k[None, None], v[None, None], padded[None], block)
    assert int(r["nblk"]) == (T - 37 + block - 1) // block
    out = _ratios(q, k, v, padded, block, ctx, mx, sm, probs)
    assert max(out.values()) <= 1.0, out
    if std == 1.0:
        assert out["ctx"] >= 0.03 and out["gate"] >= 0.03, out


@pytest.mark.parametrize("D,block,T", [(64, 128, 4096), (128, 64, 2048)])
def test_attention_bounds_refuse_a_rescale_skipped_after_block_8(D, block, T):
    """The O rescale left out from the 9th key block on (a kernel that only rescales the first 8 blocks, all that
    T <= 1024 walks at 128-key blocks) leaves the element bound and the gate on diffuse and on rising logits, while
    the correct emulation of the same rows stays inside"""
    for std, rise in ((1.0, False), (2.0, True)):
        q, k, v, padded = _long_inputs(T, D, std, rise, seed=3 * T + D)
        good, _, _, _ = _emulate_attention(q, k, v, padded, block)
        assert max(_ratios(q, k, v, padded, block, good).values()) <= 1.0
        bad, _, _, _ = _emulate_attention(q, k, v, padded, block, skip_rescale_from=8)
        out = _ratios(q, k, v, padded, block, bad)
        assert out["ctx"] > 1.0 and out["gate"] > 1.0, (std, rise, out)


# ---- tied row attention ---------------------------------------------------------------------------------------------
def _tied_qkv(B, R, C, H, std, seed, split):
    """qkv [B*R*C, 3E] fp16 (or [B*R*C, 6E] hi | lo) with summed logits of std `std`"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, R, C, 3, H, 64, generator=g, dtype=torch.float64)
    x[:, :, :, 0] *= std / math.sqrt(64 * R)
    x = x.reshape(B * R * C, 3 * 64 * H)
    if split:
        return torch.cat(kr.split16(x), 1)
    return x.half()


def _emulate_tied(qkv, key_pad, B, R, C, H, split, drop_slab=None, drop_lohi=False, p_scale=1.0, ctx_scale=1.0,
                  v_shift=0):
    """float64 emulation of tied_scores / tied_softmax / tied_pv: logits in truncating k16 steps (fp16: one accumulator
    over all rows; split: a fresh fragment per row, q_lo k_hi, q_hi k_lo, q_hi k_hi per step, then an fp32 add), the
    softmax with fp32 roundings (exp2 correctly rounded, flushed below 2^-126) and the lane / shuffle sum order, P V in
    truncating k16 steps.  Returns S [H,B,C,C], P halves [H,B,C,Cp], the fp32 probabilities and ctx halves
    [B,R,C,H,64].  Faults: drop_slab (an alignment row left out of the logits), drop_lohi (the split slab's q_lo k_hi
    pass left out), p_scale (q scaled before it is stored), ctx_scale (the accumulator scaled before the output),
    v_shift (V read from alignment row r + v_shift)."""
    _, hi, lo = kr.tied_operands(qkv, B, R, C, H, split)
    Cp = (C + 63) // 64 * 64
    S = torch.zeros(H, B, C, C, dtype=torch.float64)
    for r in range(R):
        if r == drop_slab:
            continue
        part = torch.zeros_like(S) if split else S
        for d0 in range(0, 64, 16):
            sl = slice(d0, d0 + 16)
            terms = [(hi, hi)]
            if split:
                terms = ([] if drop_lohi else [(lo, hi)]) + [(hi, lo), (hi, hi)]
            for a, b in terms:
                part = _chop(part + kr._qk(a[:, r:r + 1, :, 0, :, sl], b[:, r:r + 1, :, 1, :, sl]))
        S = _f32(S + part) if split else part
    x = S.masked_fill(kr.tied_pad(key_pad, B, C, S.device), -10000.0)
    m = x.amax(-1, keepdim=True)
    t = _f32(_f32(x - m) * LOG2E32)
    e = _f32(torch.exp2(t))
    e = torch.where(e < 2.0 ** -126, torch.zeros_like(e), e)
    lanes = torch.nn.functional.pad(e, (0, 1024 - C)).view(H, B, C, 32, 32)  # [.., i, lane]: column 32 i + lane
    acc = torch.zeros(H, B, C, 32, dtype=torch.float64)
    for i in range(32):
        acc = _f32(acc + lanes[..., i, :])
    for o in (16, 8, 4, 2, 1):
        acc = _f32(acc + acc[..., torch.arange(32) ^ o])
    inv = _f32(1.0 / acc[..., :1])
    q = _f32(_f32(e * inv) * p_scale)
    qp = torch.nn.functional.pad(q, (0, Cp - C))
    P_hi = qp.half().double()
    P_lo = _f32(qp - P_hi).half().double() if split else None
    vh = torch.roll(hi[:, :, :, 2], -v_shift, 1)
    vl = torch.roll(lo[:, :, :, 2], -v_shift, 1) if split else None
    vpad = lambda w: torch.nn.functional.pad(w, (0, 0, 0, 0, 0, Cp - C))  # noqa: E731  keys C .. Cp: zero
    vh, vl = vpad(vh), (vpad(vl) if split else None)
    out = torch.zeros(B, R, C, H, 64, dtype=torch.float64)
    for s0 in range(0, Cp, 16):
        sl = slice(s0, s0 + 16)
        terms = [(P_hi, vh)] + ([(P_lo, vh), (P_hi, vl)] if split else [])
        for a, w in terms:
            out = _chop(out + kr._pv(a[..., sl], w[:, :, sl]))
    out = _f32(out * ctx_scale)
    c_hi = out.half().double()
    c_lo = _f32(out - c_hi).half().double() if split else None
    return S, (P_hi, P_lo), q, (c_hi, c_lo)


def _tied_ratios(qkv, key_pad, B, R, C, H, split, em):
    """worst ratio of each stage and of the end-to-end checks to its kernel_refs bound"""
    S, (P_hi, P_lo), q, (c_hi, c_lo) = em
    r = kr.tied64(qkv, key_pad, B, R, C, H, split)
    sr = kr.tied_softmax64(S.float(), key_pad)
    P = P_hi if P_lo is None else P_hi + P_lo
    _, hi, lo = kr.tied_operands(qkv, B, R, C, H, split)
    pv_ref, pv_b = kr.tied_pv(P_hi[..., :C], None if P_lo is None else P_lo[..., :C], hi[:, :, :, 2],
                              None if lo is None else lo[:, :, :, 2], r["Cp"])
    ctx = c_hi if c_lo is None else c_hi + c_lo
    out = dict(logits=float(((S - r["s"]).abs() / r["lerr"]).max()),
               P=float(((P[..., :C] - sr["p"]).abs() / kr.tied_P_bound(sr, split)).max()),
               probs=float(((q - sr["p"]).abs() / kr.tied_probs_bound(sr)).max()),
               rowsum=float(((q.sum(-1) - 1).abs() / kr.tied_rowsum_bound(C)).max()),
               pv=float(((ctx - pv_ref).abs() / pv_b).max()),
               ctx=float(((ctx - r["ctx"]).abs() / kr.tied_ctx_bound(r)).max()))
    rf = (ctx - r["ctx"]).pow(2).sum((1, 2, 4)).sqrt() / r["ctx"].pow(2).sum((1, 2, 4)).sqrt()
    out["gate"] = float((rf / kr.tied_relfro_gate(r)).max())
    return out


def _tied_pad(B, C):
    pad = torch.zeros(B, C, dtype=torch.uint8)
    pad[0, C - C // 7:] = 1
    pad[B - 1, C // 3] = 1
    return pad


TIED_EMU_CASES = [(1, 33, 1.0, False), (5, 97, 1.0, False), (3, 300, 3.0, False), (2, 129, 8.0, False),
                  (1, 33, 1.0, True), (5, 97, 1.0, True), (3, 300, 3.0, True), (2, 129, 8.0, True)]


@pytest.mark.parametrize("R,C,std,split", TIED_EMU_CASES)
def test_tied_bounds_cover_an_emulated_kernel(R, C, std, split):
    """The emulated kernels on two alignments with different padded key columns stay inside every stage and
    end-to-end bound, and the bounds are not vacuous: P reaches 0.1 of its bound, and with fp16 so do P V and the
    end-to-end ctx.  (With fp32x3 the end-to-end bound is led by ex2.approx's 2^-22, which the emulation, rounding
    exp2 correctly, does not reproduce.)"""
    B, H = 2, 2
    qkv = _tied_qkv(B, R, C, H, std, seed=R * 1000 + C, split=split)
    pad = _tied_pad(B, C)
    out = _tied_ratios(qkv, pad, B, R, C, H, split, _emulate_tied(qkv, pad, B, R, C, H, split))
    print("tied emulation", R, C, std, split, {k: f"{v:.3f}" for k, v in out.items()})
    assert max(out.values()) <= 1.0, out
    assert out["P"] >= 0.1 and (split or (out["pv"] >= 0.1 and out["ctx"] >= 0.1)), out


@pytest.mark.parametrize("split", [False, True], ids=["fp16", "fp32x3"])
def test_tied_bounds_refuse_emulated_faults(split):
    """P x (1 + 2^-13) leaves the probabilities' row-sum bound; ctx x (1 + 2^-9) and V read from the next alignment
    row leave the P V bound; an alignment row's slab dropped from the logits, and with fp32x3 the slab's q_lo k_hi
    pass, leave the logit bound."""
    B, R, C, H = 2, 5, 97, 2
    qkv = _tied_qkv(B, R, C, H, 1.0, seed=3, split=split)
    pad = _tied_pad(B, C)
    ratios = lambda **f: _tied_ratios(qkv, pad, B, R, C, H, split,  # noqa: E731
                                      _emulate_tied(qkv, pad, B, R, C, H, split, **f))
    assert max(ratios().values()) <= 1.0
    assert ratios(p_scale=1 + 2.0 ** -13)["rowsum"] > 1.0
    assert ratios(ctx_scale=1 + 2.0 ** -9)["pv"] > 1.0
    assert ratios(v_shift=1)["pv"] > 1.0
    assert ratios(drop_slab=R // 2)["logits"] > 1.0
    if split:
        assert ratios(drop_lohi=True)["logits"] > 1.0


# ---- embedding prologues, mean pool, log-softmax, standalone contact pass, layer ------------------------------------
def _tokens(B, T, seed, pad=1, mask=32):
    """[B,T] residues with leading, interior and trailing pads and a few <mask>; row 1 has neither"""
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(4, 24, (B, T), generator=g)
    tok[:, 0] = 0
    tok[0, T - 3:] = pad
    tok[0, 2] = tok[0, T // 2] = mask
    if B > 2:
        tok[2, :2] = pad
        tok[2, T // 3] = pad
        tok[2, 5] = mask
    return tok


def test_positions_hand_written_example():
    tok = torch.tensor([[1, 1, 0, 5, 1, 6, 1, 7, 2, 1], [0, 5, 6, 7, 8, 9, 2, 1, 1, 1]])
    want = torch.tensor([[1, 1, 2, 3, 1, 4, 1, 5, 6, 1], [2, 3, 4, 5, 6, 7, 8, 1, 1, 1]])
    assert torch.equal(kr.positions(tok, 1), want)
    assert torch.equal(kr.positions(tok[None], 1), want[None])  # over the last dim, whatever is in front
    # another padding index shifts every position and moves the pads
    assert torch.equal(kr.positions(torch.tensor([[0, 3, 5, 3, 6]]), 3), torch.tensor([[4, 3, 5, 3, 6]]))


@pytest.mark.parametrize("token_dropout", [True, False])
def test_embed_esm2_64_matches_the_oracle(token_dropout):
    from oracle import esm2_oracle
    from oracle.weights import make_state_dict
    table = make_state_dict(0, 64, 2, seed=1)["embed_tokens.weight"].double()
    tok = _tokens(3, 40, seed=2)
    want = esm2_oracle.embed(tok, {"embed_tokens.weight": table}, token_dropout)
    got = kr.embed_esm2_64(tok, table, 1, 32, token_dropout)
    torch.testing.assert_close(got, want, atol=0, rtol=1e-15)
    assert (float(got[0, 2].abs().max()) == 0.0) == token_dropout  # a <mask> row
    assert float(got[0, -1].abs().max()) == 0.0 and float(got[1].abs().min()) > 0.0
    if token_dropout:  # row 0: 2 <mask> of 37 non-pad tokens; row 1: none
        torch.testing.assert_close(got[0, 1], table[tok[0, 1]] * 0.88 / (1 - 2 / 37), rtol=1e-15, atol=0)
        torch.testing.assert_close(got[1, 1], table[tok[1, 1]] * 0.88, rtol=1e-15, atol=0)


def test_embed_esm2_64_non_finite_scales():
    """pads only: 0 / 0, NaN everywhere (the reference multiplies the pad rows by zero); every non-pad token a <mask>:
    0.88 * 0 / 0 = NaN"""
    table = torch.randn(33, 8, generator=torch.Generator().manual_seed(0))
    tok = torch.tensor([[1, 1, 1, 1], [32, 32, 32, 1], [0, 5, 32, 1]])
    got = kr.embed_esm2_64(tok, table, 1, 32, True)
    assert bool(got[0].isnan().all()) and bool(got[1].isnan().all()) and bool(got[2].isfinite().all())
    assert bool(kr.embed_esm2_64(tok, table, 1, 32, False).isfinite().all())
    b = kr.embed_scale_bound(tok, 1, 32, True)
    assert b.shape == (3, 1, 1) and float(b[0]) == 0.0 and float(b[1]) == 0.0
    assert math.isclose(float(b[2]), kr.U32 * (4 + (1 / 3) / (2 / 3)))
    assert float(kr.embed_scale_bound(tok, 1, 32, False).abs().max()) == 0.0


@pytest.mark.parametrize("token_dropout", [True, False])
def test_embed_esm1b_64_is_the_esm2_scaling_plus_positions(token_dropout):
    from oracle import esm2_oracle
    g = torch.Generator().manual_seed(3)
    E, T = 32, 40
    table = torch.randn(33, E, generator=g, dtype=torch.float64)
    pos = torch.randn(T + 2, E, generator=g, dtype=torch.float64)
    w, b = 1 + 0.2 * torch.randn(E, generator=g, dtype=torch.float64), torch.randn(E, generator=g, dtype=torch.float64)
    tok = _tokens(3, T, seed=4)
    keep = tok.ne(1)[..., None]
    scaled = esm2_oracle.embed(tok, {"embed_tokens.weight": table}, token_dropout)
    x, pre = kr.embed_esm1b_64(tok, table, pos, None, None, 1, 32, token_dropout)
    assert torch.equal(x, pre * keep)
    p = torch.zeros(3, T, dtype=torch.long)
    for i in range(3):  # the count of non-pad tokens so far, written as a loop
        n = 0
        for t in range(T):
            n += int(tok[i, t] != 1)
            p[i, t] = n + 1 if tok[i, t] != 1 else 1
    torch.testing.assert_close(x, (scaled + pos[p]) * keep, atol=0, rtol=1e-15)
    y, pre2 = kr.embed_esm1b_64(tok, table, pos, w, b, 1, 32, token_dropout)
    assert torch.equal(pre, pre2)
    torch.testing.assert_close(y, torch.nn.functional.layer_norm(pre, (E,), w, b, 1e-5) * keep, atol=0, rtol=1e-15)
    assert float(y[0, -1].abs().max()) == 0.0


@pytest.mark.parametrize("msa_pos_dim", [None, 1, 0], ids=["E", "1", "none"])
def test_embed_msa_64_matches_the_oracle_embedding(msa_pos_dim):
    from oracle.msa_oracle import make_msa_state_dict, make_msa_tokens, msa_transformer_forward
    E, H, B, R, C = 64, 2, 2, 5, 40
    sd = make_msa_state_dict(1, E, 128, H, seed=5, msa_pos_dim=msa_pos_dim or None)
    if msa_pos_dim == 0:
        del sd["msa_position_embedding"]
    sd = {k: v.double() for k, v in sd.items()}
    tok = make_msa_tokens(B, R, C, seed=6, pad_cols=4, pad_rows_last=2)
    tok[0, 1, 3] = tok[0, 2, 0] = 1  # interior and leading pads
    # representation 0 of a one-layer model: the embedding (with no layer at all it would be the final LayerNorm's)
    want = msa_transformer_forward(sd, 1, H, tok, repr_layers=[0])["representations"][0]
    mp = sd["msa_position_embedding"][0, :, 0] if "msa_position_embedding" in sd else None  # [1024, E or 1]
    got, pre = kr.embed_msa_64(tok, sd["embed_tokens.weight"], sd["embed_positions.weight"], mp,
                               sd["emb_layer_norm_before.weight"], sd["emb_layer_norm_before.bias"], 1)
    torch.testing.assert_close(got, want, atol=1e-13, rtol=1e-13)
    assert pre.shape == (B, R, C, E) and kr.row_cond(pre, tok, 1) < 10


def test_mean_pool64_clamps_and_gives_nan_for_the_empty_slice():
    g = torch.Generator().manual_seed(7)
    x = torch.randn(6, 10, 8, generator=g)
    lengths = torch.tensor([9, 4, 0, -3, 12, 1], dtype=torch.int32)
    got = kr.mean_pool64(x, lengths)
    for b, n in enumerate([9, 4, 0, 0, 9, 1]):
        assert bool(got[b].isnan().all()) == (n == 0)
        if n:
            assert torch.equal(got[b], x[b, 1:1 + n].double().mean(0))
    assert torch.equal(got[4], x[4, 1:1 + 12].double().mean(0))  # the slice's own clamp
    bound = kr.mean_pool_bound(x, lengths)
    f32 = torch.stack([x[b, 1:1 + n].sum(0) / n for b, n in ((0, 9), (1, 4), (4, 9), (5, 1))]).double()
    ok = torch.tensor([0, 1, 4, 5])
    assert bool(((f32 - got[ok]).abs() <= bound[ok]).all()) and float(bound[ok].max()) < 1e-6


def test_log_softmax64_matches_torch_and_its_bound_holds_in_fp32():
    g = torch.Generator().manual_seed(8)
    x = (torch.rand(50, 33, generator=g) * 160 - 80)
    x[3, 5] = float("-inf")
    x[4] = float("-inf")
    x[5, 7] = 300.0  # dominant: lse ~ 0
    got = kr.log_softmax64(x)
    want = torch.log_softmax(x.double(), -1)
    fin = torch.ones(50, dtype=torch.bool)
    fin[4] = False
    torch.testing.assert_close(got[fin], want[fin], atol=1e-12, rtol=1e-13)
    assert bool(got[4].isnan().all()) and got[3, 5] == float("-inf") and float(got[5, 7]) == 0.0
    bound = kr.log_softmax_bound(x)
    live = got.isfinite()
    assert bool(((torch.log_softmax(x, -1).double() - got).abs()[live] <= bound[live]).all())
    # a fault: column 32 left out of the sum, on the rows where it carries weight
    m = x[:, :32].amax(-1, keepdim=True)
    half = ((x - m) - torch.log(torch.exp(x[:, :32] - m).sum(-1, keepdim=True))).double()
    rows = x[:, 32] > x[:, :32].amax(-1) - 5
    assert bool(rows.any()) and bool(((half - got).abs()[rows][:, :32] > bound[rows][:, :32]).all())


def test_contact_stripes_sum_to_the_reference_contact_head():
    from oracle import esm2_oracle
    from oracle.weights import make_tokens
    L, H, T = 2, 3, 40
    tokens = make_tokens([38, 20], T, seed=9)
    attn = _random_maps(L, 2, H, T, seed=10)
    g = torch.Generator().manual_seed(11)
    sd = {"contact_head.regression.weight": torch.randn(1, L * H, generator=g, dtype=torch.float64),
          "contact_head.regression.bias": torch.randn(1, generator=g, dtype=torch.float64)}
    want = esm2_oracle.contact_head(tokens, attn, sd)
    w = sd["contact_head.regression.weight"].view(L, H)
    parts = [kr.contact_stripes(attn[:, l], w[l], tokens.ne(2), 1, T - 1) for l in range(L)]
    assert parts[0][1].shape == (2, H, 38) and parts[0][2].shape == (2, H, 3, 38)
    a = kr.masked_maps(attn[:, 0], tokens.ne(2), 1, T - 1)[:, :, 1:T - 1, 1:T - 1]
    torch.testing.assert_close(parts[0][2][:, :, 2], a[:, :, 32:38].sum(-2), atol=0, rtol=1e-14)  # the partial stripe
    torch.testing.assert_close(parts[0][2][:, :, 1], a[:, :, 16:32].sum(-2), atol=0, rtol=1e-14)
    got = kr.contacts_from_partials(sum(p[0] for p in parts), torch.stack([p[1][:, :, None] for p in parts]),
                                    torch.stack([p[2] for p in parts]), w, float(sd["contact_head.regression.bias"]))
    torch.testing.assert_close(got, want, atol=1e-12, rtol=1e-12)


@pytest.mark.parametrize("E,H", [(128, 2), (144, 2)], ids=["d64", "d72"])
def test_layer64_matches_the_oracle_layer(E, H):
    from oracle import esm2_oracle
    from oracle.weights import make_state_dict
    sd = {k: v.double() for k, v in make_state_dict(1, E, H, seed=12).items()}
    g = torch.Generator().manual_seed(13)
    x = torch.randn(2, 30, E, generator=g, dtype=torch.float64)
    pad = torch.zeros(2, 30, dtype=torch.bool)
    pad[1, 21:] = True
    sd32 = {k: v.float() for k, v in sd.items()}
    want, wp = esm2_oracle.transformer_layer(x.float(), sd32, "layers.0.", H, pad, True)  # the fp32 oracle
    got, gp = kr.layer64(x, sd, "layers.0.", H, pad)
    torch.testing.assert_close(gp, wp.double(), atol=2e-6, rtol=0)
    torch.testing.assert_close(got, want.double(), atol=3e-5, rtol=0)
    assert float(gp[1, :, :, 21:].abs().max()) == 0.0


# ---- the bounds of the layer-stack stages (tests/stack_replay.py) ---------------------------------------------------
def _fp16_operands(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) * K ** -0.5).half()
    return a, w, 0.1 * torch.randn(N, generator=g)


@pytest.mark.parametrize("K", [1280, 5120])
def test_residual_bound_holds_for_fp32_and_refuses_a_scaled_update(K):
    """x + fp32(a w^T + bias) (an fp32 GEMM, then the fp32 add) stays inside residual_bound; the update scaled by
    1 + 2^-9 leaves it"""
    M, N = 192, 256
    a, w, bias = _fp16_operands(M, N, K, K)
    x = torch.randn(M, N, generator=torch.Generator().manual_seed(K + 1))
    y32 = a.float() @ w.float().t() + bias
    y, absdot = kr.gemm_exact(a, w, bias)
    want = x.double() + y
    b = kr.residual_bound(kr.gemm_acc_bound(absdot, K, y), want)
    assert float(((x + y32).double() - want).abs().div(b).max()) <= 1.0
    bad = x + y32 * (1 + 2.0 ** -9)
    assert float((bad.double() - want).abs().div(b).max()) > 1.5


def test_qkv_bound_holds_for_fp32_and_refuses_a_shifted_rotation():
    """the QKV epilogue restated in fp32 (bias, q scale, rotate-half by the [T, 32] table, fp16 output) stays inside
    qkv_bound around qkv_ref; the same with every row rotated by the next position's table row leaves it"""
    from esm_b200.model import rope_tables
    T, B, H = 64, 2, 2
    E, M = 64 * H, 2 * 64
    a, w, bias = _fp16_operands(M, 3 * E, E, 5)
    inv = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
    cos, sin = rope_tables(inv, T + 1)

    def emulate(shift):
        y = a.float() @ w.float().t() + bias
        y[:, :E] *= 0.125
        t = torch.arange(M) % T + shift
        c, s = cos[t], sin[t]
        for g0 in range(0, 2 * E, 64):
            x1, x2 = y[:, g0:g0 + 32].clone(), y[:, g0 + 32:g0 + 64].clone()
            y[:, g0:g0 + 32], y[:, g0 + 32:g0 + 64] = x1 * c - x2 * s, x2 * c + x1 * s
        return y.half()

    want, absdot = kr.qkv_ref(a, w, bias, 0.125, E, T, cos[:T], sin[:T])
    b = kr.qkv_bound(want, absdot, E)
    assert float((emulate(0).double() - want).abs().div(b).max()) <= 1.0
    assert float((emulate(1).double() - want).abs().div(b).max()) > 10


def test_replay_q_scales_are_the_references_fp32_values():
    """stack_replay.q_scale rounds the reference's double to fp32, and differs by one ulp from the fp32 expression the
    library used before at the widths and depths DESIGN.md section 4 lists"""
    import stack_replay as sr
    assert sr.q_scale(64) == 0.125 and sr.q_scale(24) == float(np.float32(24 ** -0.5))
    old = [d for d in range(2, 129, 2) if sr.q_scale(d) != float(np.float32(1) / np.sqrt(np.float32(d)))]
    assert old == [6, 18, 24, 28, 34, 58, 68, 72, 78, 82, 84, 94, 96, 102, 112, 122]
    rows = [R for R in range(1, 1025) if sr.q_scale(64, R) != float(np.float32(0.125) / np.sqrt(np.float32(R)))]
    assert len(rows) == 242 and rows[:3] == [6, 7, 17]


# ---- heads in 64-wide slots at any head width (tests/stack_replay.py pack_esm, qkv_stage) ---------------------------
# every width tests/test_gpu_stack_head_widths.py and the stage tests run, and widths that fill a slot partly (8, 40) or
# the second slot partly (66: one pair, 126: thirty-one)
SLOT_WIDTHS = [16, 24, 32, 64, 128, 8, 40, 66, 126]
SLOT_H = 3


def _slot_tables(d, T, dtype):
    """the reference's [T, d/2] tables (rotary_embedding.py:47-61) and the replay's [T, 32 slots] widening of them"""
    import stack_replay as sr
    inv = 1.0 / (10000 ** (torch.arange(0, d, 2, dtype=torch.float64) / d))
    f = torch.arange(T, dtype=torch.float64)[:, None] * inv[None]
    cos, sin = f.cos().to(dtype), f.sin().to(dtype)
    return (cos, sin) + sr.rope_slots(cos, sin, kr.head_slots(d * SLOT_H, SLOT_H))


def _slot_rotate(z, E, H, cos_s, sin_s, T):
    """the QKV epilogue's rotation (csrc/gemm_common.cuh epi_qkv_box) on a head-slot tensor z [M, 3Ea]: columns
    (c, c + 32) of every 64-wide group of q and k rotated by column 32 (group mod slots) + c of the [T, 32 slots] table"""
    slots = kr.head_slots(E, H)
    Ea = 64 * slots * H
    t = torch.arange(z.shape[0]) % T
    z = z.clone()
    for g0 in range(0, 2 * Ea, 64):
        s = (g0 // 64) % slots
        c, sn = cos_s[t][:, 32 * s:32 * s + 32], sin_s[t][:, 32 * s:32 * s + 32]
        x1, x2 = z[:, g0:g0 + 32].clone(), z[:, g0 + 32:g0 + 64].clone()
        z[:, g0:g0 + 32], z[:, g0 + 32:g0 + 64] = x1 * c - x2 * sn, x2 * c + x1 * sn
    return z


def _pack_cols(y, rows, Ea3):
    z = torch.zeros(y.shape[0], Ea3, dtype=y.dtype)
    z[:, rows] = y
    return z


@pytest.mark.parametrize("d", SLOT_WIDTHS)
def test_slot_map_is_the_head_slot_map_and_round_trips(d):
    """slot_columns, derived from the rotate-half pairing, is the map fp8_refs.head_slot states (elementwise.cuh
    head_slot); it is one to one into [0, Ea), and unpacking through slot_rows inverts packing, leaving 3 (Ea - E) padding
    columns that hold zeros"""
    import fp8_refs
    import stack_replay as sr
    H = SLOT_H
    E = d * H
    Ea = 64 * kr.head_slots(E, H) * H
    cols = kr.slot_columns(d, H)
    assert torch.equal(cols, fp8_refs.head_slot(torch.arange(E), d))
    assert cols.unique().numel() == E and int(cols.min()) >= 0 and int(cols.max()) < Ea
    rows = kr.slot_rows(d, H)
    y = torch.randn(7, 3 * E, dtype=torch.float64, generator=torch.Generator().manual_seed(d))
    z = _pack_cols(y, rows, 3 * Ea)
    assert torch.equal(z[:, rows], y)
    pad = sr.padding_columns(rows, 3 * Ea)
    assert int(pad.sum()) == 3 * (Ea - E) and bool((z[:, pad] == 0).all())
    assert torch.equal(_pack_cols(z[:, rows], rows, 3 * Ea), z)


@pytest.mark.parametrize("d", SLOT_WIDTHS)
def test_slot_rotation_is_the_reference_rotate_half(d):
    """the kernel's (c, c + 32) rotation by table column 32 slot + c on the packed heads, unpacked, equals the oracle's
    rotate-half on every q and k head bit for bit in float64 (and qkv_ref_heads' rotation); v and the padding columns
    (rotated by the replay's padding values) stay as they were"""
    import stack_replay as sr
    from oracle import esm2_oracle
    H, T = SLOT_H, 40
    E = d * H
    Ea = 64 * kr.head_slots(E, H) * H
    cos, sin, cos_s, sin_s = _slot_tables(d, T, torch.float64)
    rows = kr.slot_rows(d, H)
    M = 2 * T
    y = torch.randn(M, 3 * E, dtype=torch.float64, generator=torch.Generator().manual_seed(d + 1))
    z = _slot_rotate(_pack_cols(y, rows, 3 * Ea), E, H, cos_s, sin_s, T)
    t = torch.arange(M) % T
    want = y.clone()
    for sec in range(2):
        x = y[:, sec * E:(sec + 1) * E].view(M, H, d)
        want[:, sec * E:(sec + 1) * E] = esm2_oracle.apply_rope(x, cos[t][:, None], sin[t][:, None]).reshape(M, E)
    assert torch.equal(z[:, rows], want)
    assert bool((z[:, sr.padding_columns(rows, 3 * Ea)] == 0).all())
    # qkv_ref_heads' rotation: an identity weight and zero bias pass y through the GEMM exactly
    got, _ = kr.qkv_ref_heads(y, torch.eye(3 * E, dtype=torch.float64), torch.zeros(3 * E, dtype=torch.float64), 1.0,
                              H, T, cos, sin)
    assert torch.equal(got, want)


def test_qkv_ref_heads_is_qkv_ref_at_d64():
    from esm_b200.model import rope_tables
    T, H = 32, 3
    E = 64 * H
    a, w, bias = _fp16_operands(2 * T, 3 * E, E, 8)
    inv = 1.0 / (10000 ** (torch.arange(0, 64, 2).float() / 64))
    cos, sin = rope_tables(inv, T)
    y0, d0 = kr.qkv_ref(a, w, bias, 0.125, E, T, cos, sin)
    y1, d1 = kr.qkv_ref_heads(a, w, bias, 0.125, H, T, cos, sin)
    assert torch.equal(y0, y1) and torch.equal(d0, d1)


def _emulate_qkv(a, w, bias, d, H, T, cos_s, sin_s, cols):
    """the QKV GEMM and epilogue restated in fp32 on weights packed by the column map `cols` ([E] -> [0, Ea)): bias,
    q scale fp32(d ** -0.5), the slot rotation, fp16 output; returns the output read back through the same map"""
    import stack_replay as sr
    E = d * H
    Ea = 64 * kr.head_slots(E, H) * H
    rows = torch.cat([s * Ea + cols for s in range(3)])
    ws = torch.zeros(3 * Ea, E)
    ws[rows] = w.float()
    bs = torch.zeros(3 * Ea)
    bs[rows] = bias.float()
    y = a.float() @ ws.t() + bs
    y[:, :Ea] *= sr.q_scale(d)
    return _slot_rotate(y, E, H, cos_s, sin_s, T).half()[:, rows]


@pytest.mark.parametrize("d", SLOT_WIDTHS)
def test_qkv_heads_bound_holds_and_refuses_a_wrong_slot_or_table_column(d):
    """the fp32 restatement stays inside qkv_bound around qkv_ref_heads (K = E); rotating every pair by the neighbouring
    table column leaves it, and at two slots per head (d > 64) so does a map that sends each pair to the head's other
    slot"""
    import stack_replay as sr
    H, T = SLOT_H, 48
    E = d * H
    a, w, bias = _fp16_operands(2 * T, 3 * E, E, d + 2)
    cos, sin, cos_s, sin_s = _slot_tables(d, T, torch.float32)
    want, absdot = kr.qkv_ref_heads(a, w, bias, sr.q_scale(d), H, T, cos, sin)
    b = kr.qkv_bound(want, absdot, E)
    ratio = lambda got: float((got.double() - want).abs().div(b).max())  # noqa: E731
    cols = kr.slot_columns(d, H)
    assert ratio(_emulate_qkv(a, w, bias, d, H, T, cos_s, sin_s, cols)) <= 1.0
    shifted = lambda t: torch.cat([t[:, 1:], t[:, -1:]], 1)  # noqa: E731  column p reads column p + 1
    assert ratio(_emulate_qkv(a, w, bias, d, H, T, shifted(cos_s), shifted(sin_s), cols)) > 10
    if kr.head_slots(E, H) == 2:
        other = cols + torch.where((cols // 64) % 2 == 0, 64, -64)  # the head's other slot, same columns
        assert ratio(_emulate_qkv(a, w, bias, d, H, T, cos_s, sin_s, other)) > 10


# ---- the column attention maps (tests/stack_replay.py column_query_rows, column_zero_stage, qrows) -------------------
def test_column_query_rows_are_every_row_of_a_live_column():
    import stack_replay as sr
    cpad = torch.tensor([[False, False, True], [True, True, True], [True, False, True]])
    want = torch.tensor([[True] * 3, [False] * 3, [True] * 3])
    assert torch.equal(sr.column_query_rows(cpad), want)


def test_column_zero_stage_refuses_a_padded_key_or_a_dead_column_with_probability():
    import stack_replay as sr
    cpad = torch.tensor([[False, True], [True, True]])
    p = torch.zeros(2, 1, 2, 2)
    p[0, 0, :, 0] = 1.0
    sr.column_zero_stage("maps", p, cpad)
    for idx in ((0, 0, 1, 1), (1, 0, 0, 0)):
        bad = p.clone()
        bad[idx] = 2.0 ** -126
        with pytest.raises(AssertionError):
            sr.column_zero_stage("maps", bad, cpad)


def test_attention_stage_f16_checks_the_padded_query_rows_it_is_given():
    """float64 column maps rounded to fp32 pass attention_stage_f16 at every query row of the live columns; the padded
    query rows zeroed (esm2.py's stacked-map rule, wrong for the column attention) fail it, and go unseen with the
    default selection of the valid rows only"""
    import stack_replay as sr
    N, R, H = 3, 70, 2
    g = torch.Generator().manual_seed(11)
    qkv = torch.randn(N * R, 3 * 64 * H, generator=g)
    qkv[:, :64 * H] *= 0.25
    qkv = qkv.half()
    cpad = torch.zeros(N, R, dtype=torch.bool)
    cpad[1, 40:] = True
    cpad[2] = True
    q, k, v = (sr._heads(qkv, N, R, H, i) for i in range(3))
    r = kr.attention64(q, k, v, cpad, 64)
    ctx = r["ctx"].transpose(1, 2).reshape(N * R, 64 * H).half()
    probs = r["p"].float()
    qrows = sr.column_query_rows(cpad)
    worst = {}
    sr.attention_stage_f16(worst, qkv, ctx, cpad, N, R, H, probs, blocks=(64, 128), qrows=qrows)
    assert worst["probs"] <= 1.0 and worst["rowsum"] <= 1.0, worst
    bad = probs.clone()
    bad[1, :, 40:] = 0.0
    sr.attention_stage_f16({}, qkv, ctx, cpad, N, R, H, bad, blocks=(64, 128))  # valid rows only: unseen
    worst = {}
    sr.attention_stage_f16(worst, qkv, ctx, cpad, N, R, H, bad, blocks=(64, 128), qrows=qrows)
    assert worst["probs"] > 1e3 and worst["rowsum"] > 1e3, worst
