"""CPU: the float64 references of tests/kernel_refs.py that the kernel-level GPU tests compare against.

  * the contact partials, summed, give the reference contact head (oracle.esm2_oracle.contact_head) on random maps, and
    each partial is the sum over its own 32-wide quarter (a swapped quarter or tile index in the reference fails here);
  * the per-model GEMM launch table reproduces the packed layer size the library reports and the shapes of the models'
    own modules;
  * the erf-GELU bound holds for an fp32 restatement of the epilogue's formula."""
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
