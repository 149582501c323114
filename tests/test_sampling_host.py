"""CPU: Gibbs sampling (esm_b200.sampling) without a GPU. The numpy restatement of Philox4x32-10 against the toolkit's
known answers, the uniform map, the order and block partition of a sweep, a Gumbel-max frequency check of the
restatement, every refusal of gibbs raised before any launch, the command line's parser and refusal of random-init
models, and the new C ABI symbols."""
import argparse
import json
import os
import re
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # sampling_refs

import sampling_refs as sr  # noqa: E402

ROOT = os.path.dirname(HERE)


# ---- the random stream ------------------------------------------------------------------------------------------
def test_philox_matches_the_toolkit_known_answers(golden_dir):
    with open(os.path.join(golden_dir, "philox4x32_10.json")) as f:
        cases = json.load(f)["cases"]
    assert len(cases) >= 5
    counters = {tuple(c["counter"]) for c in cases}
    assert (0, 0, 0, 0) in counters and (2 ** 32 - 1,) * 4 in counters
    for c in cases:
        seed = c["key"][0] | (c["key"][1] << 32)
        got = [int(v) for v in sr.philox4x32_10(*c["counter"], seed)]
        assert got == c["out"], c


def test_philox_is_vectorised_like_the_scalar_call():
    a = sr.philox4x32_10(3, np.arange(5), 7, 1, 2 ** 63 + 5)
    for j in range(5):
        s = sr.philox4x32_10(3, j, 7, 1, 2 ** 63 + 5)
        assert [int(w[j]) for w in a] == [int(w) for w in s]


def test_uniform_map_stays_in_the_open_interval_and_is_exact_below_one_half():
    r = np.array([0, 255, 256, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 256, 2 ** 32 - 1], dtype=np.uint64)
    u = sr.uniform(r)
    assert u.dtype == np.float32 and bool(((u > 0) & (u < 1)).all())
    assert u[0] == np.float32(2.0 ** -25) and u[1] == u[0]
    assert u[2] == np.float32(3 * 2.0 ** -25)
    assert float(u[3]) == ((2 ** 23 - 1) + 0.5) * 2.0 ** -24  # the largest value below 1/2, exact
    assert float(u[4]) == 0.5  # (2^23 + 0.5) 2^-24 rounded toward zero
    assert float(u[-1]) == 1 - 2.0 ** -24


# ---- order and partition ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,block", [(1, 1), (7, 3), (10, 10), (10, 64), (33, 8), (256, 8)])
def test_every_position_once_per_sweep_and_the_block_sizes(n, block):
    g = np.random.default_rng(n)
    positions = np.sort(g.choice(1000, n, replace=False))
    k = min(block, n)
    for chain, sweep, seed in [(0, 0, 0), (5, 3, 2 ** 64 - 1), (2 ** 32 - 1, 7, 12345)]:
        blocks = sr.sweep_blocks(positions, chain, sweep, seed, block)
        assert len(blocks) == -(-n // k)
        assert [len(b) for b in blocks[:-1]] == [k] * (len(blocks) - 1)
        assert len(blocks[-1]) == n - k * (len(blocks) - 1)
        assert sorted(np.concatenate(blocks).tolist()) == positions.tolist()
    steps = 3 * len(sr.sweep_blocks(positions, 0, 0, 0, block))
    assert steps == 3 * -(-n // k)


def test_orders_differ_between_chains_sweeps_and_seeds():
    positions = np.arange(40)
    base = np.concatenate(sr.sweep_blocks(positions, 0, 0, 0, 1))
    for chain, sweep, seed in [(1, 0, 0), (0, 1, 0), (0, 0, 1)]:
        assert not np.array_equal(np.concatenate(sr.sweep_blocks(positions, chain, sweep, seed, 1)), base)
    keys = sr.order_keys(positions, np.arange(4), 0, 9)
    assert keys.shape == (4, 40) and np.array_equal(keys % (1 << 20), np.broadcast_to(positions, (4, 40)))


def test_gumbel_max_frequencies_of_the_restatement():
    """20,000 draws of one row over distinct steps: chi-square against softmax(z)."""
    from scipy.stats import chisquare
    z = np.linspace(-2.0, 1.5, 20).astype(np.float32)
    n = 20000
    words = sr.philox4x32_10(np.arange(n)[:, None], 3, 17, np.arange(1, 6)[None, :], 4242)
    u = sr.uniform(np.stack(words, -1).reshape(n, 20))
    _, a = sr.gumbel_max_f64(np.broadcast_to(z, (n, 20)), u)
    p = np.exp(sr.log_softmax_f64(z))
    counts = np.bincount(a, minlength=20)
    stat, pval = chisquare(counts, p * n)
    print(f"restated Gumbel-max chi-square {stat:.2f}, p = {pval:.3g}")
    assert pval > 1e-3
    assert np.array_equal(sr.uniforms(5, [3], [17], 4242, 20)[0], u[5])


# ---- refusals, before any launch: CPU-resident models would raise Esmb200Error at the first launch ---------------
def _esm2():
    from esm_b200 import ESM2
    return ESM2(num_layers=1, embed_dim=128, attention_heads=2).eval()


def _tokens(model, seq="MKTAYIAKQR"):
    return model.alphabet.get_batch_converter()([("p", seq)])[2]


def test_a_valid_call_on_a_cpu_model_reaches_the_launch():
    from esm_b200 import _lib, sampling
    model = _esm2()
    with pytest.raises(_lib.Esmb200Error):
        sampling.gibbs(model, _tokens(model), positions=[0, 3], chains=2, block=2, seed=2 ** 64 - 1)


REFUSALS = {
    "msa": ({}, "MSA Transformer"),
    "padding": ({}, "padding"),
    "no_cls": ({}, "<cls>"),
    "one_residue": ({}, "at least 2 residues"),
    "mask_fixed": ({"positions": [0, 1]}, "<mask>"),
    "empty": ({"positions": []}, "empty"),
    "negative": ({"positions": [-1]}, r"\[0, 10\)"),
    "beyond": ({"positions": [10]}, r"\[0, 10\)"),
    "repeated": ({"positions": [2, 2]}, "distinct"),
    "float_positions": ({"positions": [1.0]}, "integers"),
    "block0": ({"block": 0}, "block"),
    "sweeps0": ({"sweeps": 0}, "sweeps"),
    "chains0": ({"chains": 0}, "chains"),
    "chains_float": ({"chains": 2.0}, "chains"),
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
    from esm_b200 import MSATransformer, sampling
    model = _esm2()
    tokens = _tokens(model)
    kwargs, msg = REFUSALS[case]
    if case == "msa":
        args = argparse.Namespace(layers=1, embed_dim=128, ffn_embed_dim=512, attention_heads=2, dropout=0.0,
                                  attention_dropout=0.0, activation_dropout=0.0, max_tokens_per_msa=2 ** 14,
                                  max_tokens=2 ** 14, max_positions=1024, embed_positions_msa=True)
        model = MSATransformer(args, "msa_transformer").eval()
        tokens = tokens[:, None]
    elif case == "padding":
        tokens = torch.cat([tokens, torch.tensor([[model.padding_idx]])], 1)
    elif case == "no_cls":
        tokens = tokens[:, 1:]
    elif case == "one_residue":
        tokens = _tokens(model, "M")
    elif case == "mask_fixed":
        tokens = tokens.clone()
        tokens[0, 5] = model.mask_idx  # residue 4, not designable
    with pytest.raises(ValueError, match=msg):
        sampling.gibbs(model, tokens, **kwargs)


def test_the_framing_checks_are_shared_with_the_jacobian():
    from esm_b200 import jacobian, sampling
    model = _esm2()
    tokens = _tokens(model, "M")
    with pytest.raises(ValueError, match="the categorical Jacobian needs at least 2 residues, got 1"):
        jacobian.categorical_jacobian(model, tokens)
    with pytest.raises(ValueError, match="sampling needs at least 2 residues, got 1"):
        sampling.gibbs(model, tokens)


def test_a_mask_at_a_designable_position_is_accepted():
    from esm_b200 import _lib, sampling
    model = _esm2()
    tokens = torch.tensor([[model.cls_idx] + [model.mask_idx] * 6 + [model.eos_idx]])
    with pytest.raises(_lib.Esmb200Error):  # reaches the launch
        sampling.gibbs(model, tokens, sweeps=2, block=3)


# ---- the command line -------------------------------------------------------------------------------------------
def test_cli_parser():
    from esm_b200 import sample_cli, variants
    p = sample_cli.create_parser()
    a = p.parse_args(["esm2_t33_650M_UR50D", "--length", "50", "--out", "s.fasta"])
    assert a.length == 50 and a.sequence is None and a.positions is None and str(a.out) == "s.fasta"
    assert (a.chains, a.sweeps, a.block, a.temperature, a.seed) == (1, 1, 1, 1.0, 0)
    assert a.max_tokens == variants.DEFAULT_MAX_TOKENS and a.precision == "fp16" and not a.cpu_offload
    a = p.parse_args(["m.pt", "--sequence", "MKTAYIAKQR", "--positions", "1-3,7, 9-10", "--chains", "4", "--sweeps",
                      "2", "--block", "3", "--temperature", "0.5", "--seed", "18446744073709551615", "--max-tokens",
                      "4096", "--precision", "fp8", "--cpu-offload", "--out", "o.fa"])
    assert a.sequence == "MKTAYIAKQR" and a.positions == [0, 1, 2, 6, 8, 9]
    assert (a.chains, a.sweeps, a.block, a.temperature, a.seed) == (4, 2, 3, 0.5, 2 ** 64 - 1)
    assert a.max_tokens == 4096 and a.precision == "fp8" and a.cpu_offload
    bad = [
        ["m.pt", "--out", "o.fa"],                                        # neither start
        ["m.pt", "--sequence", "MK", "--length", "5", "--out", "o.fa"],   # both starts
        ["m.pt", "--length", "5"],                                        # no --out
        ["m.pt", "--length", "0", "--out", "o.fa"],
        ["m.pt", "--length", "5", "--positions", "0", "--out", "o.fa"],   # 1-based
        ["m.pt", "--length", "5", "--positions", "4-2", "--out", "o.fa"],
        ["m.pt", "--length", "5", "--positions", "a", "--out", "o.fa"],
        ["m.pt", "--length", "5", "--chains", "0", "--out", "o.fa"],
        ["m.pt", "--length", "5", "--block", "0", "--out", "o.fa"],
        ["m.pt", "--length", "5", "--precision", "bf16", "--out", "o.fa"],
    ]
    for argv in bad:
        with pytest.raises(SystemExit):
            p.parse_args(argv)


def test_cli_refuses_a_random_init_model(tmp_path, monkeypatch):
    from esm_b200 import sample_cli
    monkeypatch.setenv("ESMB200_ALLOW_RANDOM_INIT", "1")
    out = tmp_path / "s.fasta"
    args = sample_cli.create_parser().parse_args(["esm2_t6_8M_UR50D", "--length", "20", "--out", str(out)])
    with pytest.warns(UserWarning):
        with pytest.raises(RuntimeError, match="random-init"):
            sample_cli.run(args)
    assert not out.exists()


# ---- the C ABI --------------------------------------------------------------------------------------------------
def test_symbols_are_declared_and_exported_at_abi_version_4():
    from esm_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "esmb200.h")).read(), flags=re.S)
    for name in ("esmb200_sample_order", "esmb200_sample_rows"):
        assert re.search(rf"\b{name}\s*\(", text), name
        assert name in _lib.EXPORTS
    assert _lib.load().esmb200_abi_version() == 4


def test_sampler_entry_points_check_their_arguments_before_any_launch():
    """Every refusal returns ESMB200_EINVAL with no device: argument checks come before any CUDA call."""
    from esm_b200 import _lib
    lib = _lib.load()
    p = 16  # any non-null address: never dereferenced on a refusal
    order = lambda *a: lib.esmb200_sample_order(*a)
    assert order(p, 0, 1, 0, 0, 0, p, None) == -1                 # n == 0
    assert order(p, 4, -1, 0, 0, 0, p, None) == -1                # n_chains < 0
    assert order(p, 4, 1, 2 ** 32, 0, 0, p, None) == -1           # chain0 + n_chains > 2^32
    assert order(p, 4, 1, -1, 0, 0, p, None) == -1
    assert order(p, 4, 1, 0, 2 ** 32, 0, p, None) == -1           # sweep >= 2^32
    assert order(p, 4, 1, 0, -1, 0, p, None) == -1
    assert order(p, 4, 0, 0, 0, 0, p, None) == 0                  # no chains: nothing launched
    rows = lambda **kw: lib.esmb200_sample_rows(*{**dict(
        logits=p, ld=33, n=8, set=p, n_set=21, tau=1.0, seed=0, step=0, chain0=0, per=2, ent=p, tok=p, stride=40,
        R=4, C=10, logq=p, logp=None, lstride=0, stream=None), **kw}.values())
    for kw in [dict(n=-1), dict(per=0), dict(n=7), dict(n_set=0), dict(n_set=33), dict(ld=0), dict(tau=0.0),
               dict(tau=-1.0), dict(tau=float("inf")), dict(tau=float("nan")), dict(R=0), dict(C=1),
               dict(stride=39), dict(step=2 ** 32), dict(step=-1), dict(chain0=2 ** 32 - 3), dict(chain0=-1),
               dict(logp=p, lstride=0), dict(logits=None), dict(set=None), dict(ent=None), dict(tok=None),
               dict(logq=None)]:
        assert rows(**kw) == -1, kw
    assert rows(n=0) == 0
