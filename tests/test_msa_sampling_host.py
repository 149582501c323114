"""CPU: alignment sampling from the MSA Transformer (esm_b200.sampling.msa_gibbs) without a GPU. The restatement of the
20-bit visiting order and block partition, every refusal of msa_gibbs raised before any launch, a valid call reaching
the launch, and the command line's parser and designable entries."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # sampling_refs

import sampling_refs as sr  # noqa: E402


# ---- order and partition ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,block", [(1, 1), (7, 3), (100, 100), (100, 512), (333, 17), (4096, 205)])
def test_every_entry_once_per_sweep_and_the_block_sizes(n, block):
    g = np.random.default_rng(n)
    entries = np.sort(g.choice(1 << 20, n, replace=False))
    entries[-1] = (1 << 20) - 1
    entries = np.unique(entries)
    n = len(entries)
    k = min(block, n)
    for chain, sweep, seed in [(0, 0, 0), (5, 3, 2 ** 64 - 1), (2 ** 32 - 1, 7, 12345)]:
        blocks = sr.sweep_blocks(entries, chain, sweep, seed, block)
        assert len(blocks) == -(-n // k)
        assert [len(b) for b in blocks[:-1]] == [k] * (len(blocks) - 1)
        assert len(blocks[-1]) == n - k * (len(blocks) - 1)
        assert sorted(np.concatenate(blocks).tolist()) == entries.tolist()


def test_the_order_is_the_sequence_order_when_both_keys_apply():
    """x dominates the key, so the order is x ascending with ties to the smaller entry: for the residue indices of a
    protein (below 2^16) it is the order of any key x * 2^b + p with 2^b above them."""
    positions = np.random.default_rng(3).choice(65535, 300, replace=False)
    for chain, sweep, seed in [(0, 0, 0), (9, 4, 2 ** 63 + 11)]:
        a = np.concatenate(sr.sweep_blocks(positions, chain, sweep, seed, 7))
        x = sr.philox4x32_10(sweep, chain, positions, 0, seed)[0].astype(np.int64)
        assert np.array_equal(a, positions[np.lexsort((positions, x))])
        assert np.array_equal(a, np.sort(x * 65536 + positions) % 65536)


def test_entry_index_and_uniforms():
    r, j = sr.entry_token([0, 5, 6, 13], 7)
    assert r.tolist() == [0, 0, 1, 2] and j.tolist() == [1, 6, 1, 2]
    u = sr.uniforms(4, [3], [17], 4242, 20)
    words = sr.philox4x32_10(4, 3, 17, np.arange(1, 6), 4242)  # 4 arrays of 5: the 20 uniforms of one row
    assert np.array_equal(u[0], sr.uniform(np.stack(words, 1).reshape(-1)))
    u32 = sr.uniforms(4, [3, 3], [17, 18], 4242, 32)
    assert u32.shape == (2, 32) and np.array_equal(u32[0, :20], u[0]) and not np.array_equal(u32[0], u32[1])


# ---- refusals, before any launch: CPU-resident models would raise Esmb200Error at the first launch ---------------
def _msa_model(max_positions=1024):
    import argparse
    from esm_b200 import MSATransformer
    args = argparse.Namespace(layers=1, embed_dim=128, ffn_embed_dim=512, attention_heads=2, dropout=0.0,
                              attention_dropout=0.0, activation_dropout=0.0, max_tokens_per_msa=2 ** 14,
                              max_tokens=2 ** 14, max_positions=max_positions, embed_positions_msa=True)
    return MSATransformer(args, "msa_transformer").eval()


def _alignment(model, R=3, C=9):
    g = torch.Generator().manual_seed(R * 100 + C)
    t = torch.randint(4, 24, (1, R, C), generator=g)
    t[0, :, 0] = model.cls_idx
    t[0, -1, -1] = model.alphabet.get_idx("-")
    return t


def test_a_valid_call_on_a_cpu_model_reaches_the_launch():
    from esm_b200 import _lib, sampling
    model = _msa_model()
    tokens = _alignment(model)
    des = torch.zeros((3, 8), dtype=torch.bool)
    des[1:, 2:5] = True
    tokens[0, 2, 3] = model.mask_idx  # (2, 2) is designable
    with pytest.raises(_lib.Esmb200Error):
        sampling.msa_gibbs(model, tokens, designable=des, chains=2, block=2, seed=2 ** 64 - 1, gaps=False)
    appended = torch.cat([tokens, torch.full((1, 2, 9), model.mask_idx)], 1)
    appended[0, 3:, 0] = model.cls_idx
    with pytest.raises(_lib.Esmb200Error):
        sampling.msa_gibbs(model, appended, sweeps=2, block=5)


REFUSALS = {
    "sequence_model": ({}, r"sampling\.gibbs"),
    "not_a_model": ({}, "MSATransformer"),
    "float_tokens": ({}, "integer"),
    "two_alignments": ({}, r"one alignment \[1, R, C\]"),
    "two_dims": ({}, r"one alignment \[1, R, C\]"),
    "pad": ({}, "<pad>"),
    "eos": ({}, "<eos>"),
    "no_cls": ({}, "<cls>"),
    "one_column": ({}, "C >= 2"),
    "too_many_rows": ({}, "at most 1024 rows"),
    "too_many_columns": ({}, "max_positions"),
    "too_many_entries": ({}, r"at most 2\^20 residue entries"),
    "mask_fixed": ({"designable": "cols0"}, "<mask>"),
    "designable_shape": ({"designable": torch.ones((3, 9), dtype=torch.bool)}, r"designable .*\[3, 8\]"),
    "designable_dtype": ({"designable": torch.ones((3, 8), dtype=torch.int64)}, "designable must be a bool"),
    "designable_none_true": ({"designable": torch.zeros((3, 8), dtype=torch.bool)}, "at least one True"),
    "block0": ({"block": 0}, "block"),
    "sweeps0": ({"sweeps": 0}, "sweeps"),
    "chains0": ({"chains": 0}, "chains"),
    "chains_float": ({"chains": 2.0}, "chains"),
    "chains_over_2_32": ({"chains": 2 ** 32 + 1}, "at most 2"),
    "steps_over_2_32": ({"sweeps": 2 ** 32, "block": 1}, r"sweeps \* ceil\(\|designable\| / block\)"),
    "tau0": ({"temperature": 0.0}, "temperature"),
    "tau_neg": ({"temperature": -1.0}, "temperature"),
    "tau_nan": ({"temperature": float("nan")}, "temperature"),
    "tau_inf": ({"temperature": float("inf")}, "temperature"),
    "tau_fp32_zero": ({"temperature": 1e-60}, "fp32"),
    "seed_neg": ({"seed": -1}, "seed"),
    "seed_big": ({"seed": 2 ** 64}, "seed"),
    "seed_float": ({"seed": 1.5}, "seed"),
}


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_refusals_raise_value_error_before_any_launch(case):
    from esm_b200 import ESM2, sampling
    model = _msa_model()
    tokens = _alignment(model)
    kwargs, msg = REFUSALS[case]
    kwargs = dict(kwargs)
    if case == "sequence_model":
        model = ESM2(num_layers=1, embed_dim=128, attention_heads=2).eval()
        tokens = model.alphabet.get_batch_converter()([("p", "MKTAYIAKQR")])[2]
    elif case == "not_a_model":
        model = torch.nn.Linear(2, 2)
    elif case == "float_tokens":
        tokens = tokens.float()
    elif case == "two_alignments":
        tokens = torch.cat([tokens, tokens])
    elif case == "two_dims":
        tokens = tokens[0]
    elif case == "pad":
        tokens[0, 2, 8] = model.padding_idx
    elif case == "eos":
        tokens[0, 0, 8] = model.eos_idx
    elif case == "no_cls":
        tokens[0, 1, 0] = 5
    elif case == "one_column":
        tokens = tokens[:, :, :1]
    elif case == "too_many_rows":
        tokens = _alignment(model, R=1025, C=2)
    elif case == "too_many_columns":
        tokens = _alignment(model, R=1, C=1025)
    elif case == "too_many_entries":
        model = _msa_model(max_positions=1100)  # 1024 rows of 1025 residues: one entry index past 20 bits
        tokens = _alignment(model, R=1024, C=1026)
    elif case == "mask_fixed":
        des = torch.zeros((3, 8), dtype=torch.bool)
        des[:, 0] = True
        kwargs["designable"] = des
        tokens[0, 1, 2] = model.mask_idx  # entry (1, 1): fixed
    with pytest.raises(ValueError, match=msg):
        sampling.msa_gibbs(model, tokens, **kwargs)


def test_the_largest_alignment_is_accepted():
    """R = 1024 and C = max_positions: every entry index is below 2^20, and the call reaches the launch."""
    from esm_b200 import _lib, sampling
    model = _msa_model()
    with pytest.raises(_lib.Esmb200Error):
        sampling.msa_gibbs(model, _alignment(model, R=1024, C=1024), block=4096)


def test_gibbs_keeps_its_refusal_of_the_msa_transformer():
    from esm_b200 import sampling
    model = _msa_model()
    with pytest.raises(ValueError, match="gibbs samples ESM-2, ESM-1b and ESM-1v; the MSA Transformer is not supported"):
        sampling.gibbs(model, _alignment(model))


def test_the_drawable_tokens():
    from esm_b200 import jacobian, sampling
    model = _msa_model()
    a = model.alphabet
    assert sampling._drawable(model, False) == [a.get_idx(c) for c in jacobian.AMINO_ACIDS] == list(range(4, 24))
    assert sampling._drawable(model, True) == list(range(4, 24)) + [30] and a.get_tok(30) == "-"


# ---- the command line -------------------------------------------------------------------------------------------
def test_cli_parser():
    from esm_b200 import sample_msa_cli, variants
    p = sample_msa_cli.create_parser()
    a = p.parse_args(["esm_msa1b_t12_100M_UR50S", "--msa", "in.a3m", "--out", "d"])
    assert str(a.msa) == "in.a3m" and str(a.out) == "d" and a.msa_samples is None
    assert a.rows is None and a.columns is None and a.append_rows == 0 and a.gaps
    assert (a.chains, a.sweeps, a.block, a.temperature, a.seed) == (1, 1, 1, 1.0, 0)
    assert a.max_tokens == variants.DEFAULT_MAX_TOKENS and a.precision == "fp16"
    a = p.parse_args(["m.pt", "--msa", "x.a3m", "--msa-samples", "64", "--rows", "1-3", "--columns", "5-8,12",
                      "--append-rows", "4", "--chains", "8", "--sweeps", "2", "--block", "30", "--temperature", "0.5",
                      "--seed", "18446744073709551615", "--no-gaps", "--max-tokens", "4096", "--precision", "fp32x3",
                      "--out", "o"])
    assert a.msa_samples == 64 and a.rows == [0, 1, 2] and a.columns == [4, 5, 6, 7, 11] and a.append_rows == 4
    assert (a.chains, a.sweeps, a.block, a.temperature, a.seed) == (8, 2, 30, 0.5, 2 ** 64 - 1)
    assert not a.gaps and a.max_tokens == 4096 and a.precision == "fp32x3"
    bad = [
        ["m.pt", "--out", "d"],                                           # no --msa
        ["m.pt", "--msa", "x.a3m"],                                       # no --out
        ["m.pt", "--msa", "x.a3m", "--rows", "0", "--out", "d"],          # 1-based
        ["m.pt", "--msa", "x.a3m", "--columns", "4-2", "--out", "d"],
        ["m.pt", "--msa", "x.a3m", "--append-rows", "-1", "--out", "d"],
        ["m.pt", "--msa", "x.a3m", "--msa-samples", "0", "--out", "d"],
        ["m.pt", "--msa", "x.a3m", "--chains", "0", "--out", "d"],
        ["m.pt", "--msa", "x.a3m", "--precision", "fp8", "--out", "d"],
    ]
    for argv in bad:
        with pytest.raises(SystemExit):
            p.parse_args(argv)


def test_cli_designable_entries():
    from esm_b200.sample_msa_cli import designable_mask
    assert bool(designable_mask(3, 5, 0, None, None).all())
    m = designable_mask(3, 5, 2, None, None)  # appended rows only
    assert m.shape == (5, 5) and not bool(m[:3].any()) and bool(m[3:].all())
    m = designable_mask(3, 5, 2, [0], [1, 2])  # query columns 2-3, and the appended rows in full
    want = torch.zeros((5, 5), dtype=torch.bool)
    want[0, 1:3] = True
    want[3:] = True
    assert torch.equal(m, want)
    m = designable_mask(3, 5, 0, None, [4])
    assert torch.equal(m, torch.tensor([[False] * 4 + [True]] * 3))
    m = designable_mask(3, 5, 1, [1, 3], None)
    assert torch.equal(m.any(1), torch.tensor([False, True, False, True]))
    for rows, cols in [([3], None), (None, [5])]:
        with pytest.raises(ValueError, match="outside the alignment"):
            designable_mask(3, 5, 0, rows, cols)


def test_cli_refuses_a_random_init_model(tmp_path, monkeypatch):
    from esm_b200 import sample_msa_cli
    monkeypatch.setenv("ESMB200_ALLOW_RANDOM_INIT", "1")
    (tmp_path / "in.a3m").write_text(">q\nMKTAYIAKQR\n>h\nMK-AYLAKQR\n")
    out = tmp_path / "out"
    args = sample_msa_cli.create_parser().parse_args(["esm_msa1b_t12_100M_UR50S", "--msa", str(tmp_path / "in.a3m"),
                                                      "--out", str(out)])
    with pytest.warns(UserWarning):
        with pytest.raises(RuntimeError, match="random-init"):
            sample_msa_cli.run(args)
    assert not out.exists()
