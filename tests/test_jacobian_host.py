"""CPU: the categorical Jacobian (esm_b200.jacobian) without a GPU. The float64 definition of the contact map against
a brute-force evaluation, every refusal of the Python API raised before any launch, the command line's parser and
refusal of random-init models, and the C ABI's new entry points and pinned scratch sizes."""
import argparse
import os
import re
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # jacobian_refs

from jacobian_refs import contacts_brute_force, contacts_f64, contacts_f64_chunked  # noqa: E402

ROOT = os.path.dirname(HERE)


@pytest.mark.parametrize("L", [2, 3, 5])
def test_definition_matches_brute_force(L):
    g = torch.Generator().manual_seed(L)
    jac = torch.randn((L, 20, L, 20), generator=g, dtype=torch.float64) * 8
    jac += torch.randn((1, 1, L, 20), generator=g, dtype=torch.float64) * 50  # a wild-type-like offset per (j, b)
    want = contacts_brute_force(jac)
    got = contacts_f64(jac)
    assert got.shape == (L, L)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12 * float(want.abs().max()))
    assert torch.equal(got, got.T) and bool((got.diagonal() == 0).all())


@pytest.mark.parametrize("L", [2, 5, 17])
def test_chunked_reference_matches_the_definition(L):
    """contacts_f64_chunked, which the GPU test past 2^31 elements gates against, equals contacts_f64 for any slab size,
    with a large term constant along each axis in turn; its max N and max|J| are those of the whole J."""
    g = torch.Generator().manual_seed(50 + L)
    jac = torch.randn((L, 20, L, 20), generator=g) * 8
    for shape in ([1, 1, L, 20], [1, 20, L, 20], [L, 1, L, 20], [L, 20, 1, 20], [L, 20, L, 1]):
        jac += torch.randn(shape, generator=g) * 800
    want = contacts_f64(jac)
    jc = jac.double()
    for axis in range(4):
        jc = jc - jc.mean(axis, keepdim=True)
    nmax = float(jc.pow(2).sum((1, 3)).sqrt().max())
    for rows in (1, 8, L):
        got, n, j = contacts_f64_chunked(jac, rows)
        assert got.dtype == torch.float64 and got.shape == (L, L)
        assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max()), rows
        assert abs(n - nmax) <= 1e-12 * nmax and j == float(jac.abs().max())
        assert torch.equal(got, got.T) and bool((got.diagonal() == 0).all())


def test_definition_of_an_all_zero_jacobian_is_nan_off_the_diagonal():
    c = contacts_f64(torch.zeros((3, 20, 3, 20)))
    off = ~torch.eye(3, dtype=torch.bool)
    assert bool(c[off].isnan().all()) and bool((c.diagonal() == 0).all())


def test_amino_acids_are_the_alphabet_tokens_4_to_23():
    from esm_b200 import Alphabet, jacobian
    alphabet = Alphabet.from_architecture("ESM-1b")
    assert jacobian.AMINO_ACIDS == "LAGVSERTIDPKQNFYMHWC"
    assert [alphabet.get_idx(c) for c in jacobian.AMINO_ACIDS] == list(range(4, 24))


# ---- refusals, before any launch: CPU-resident models would raise Esmb200Error at the first launch ---------------
def _esm2():
    from esm_b200 import ESM2
    return ESM2(num_layers=1, embed_dim=128, attention_heads=2).eval()


def _esm1b(max_positions=1024):
    from esm_b200 import ProteinBertModel
    args = argparse.Namespace(arch="roberta_large", layers=1, embed_dim=128, ffn_embed_dim=512, attention_heads=2,
                              max_positions=max_positions, emb_layer_norm_before=True, token_dropout=True)
    return ProteinBertModel(args, "roberta_large").eval()


def _tokens(model, seq="MKTAYIAKQR"):
    return model.alphabet.get_batch_converter()([("p", seq)])[2]


def test_a_valid_call_on_a_cpu_model_reaches_the_launch():
    from esm_b200 import _lib, jacobian
    model = _esm2()
    with pytest.raises(_lib.Esmb200Error):
        jacobian.categorical_jacobian(model, _tokens(model))


@pytest.mark.parametrize("case", ["msa", "fp8", "batch", "1d", "3d", "float", "padding", "no_cls", "no_eos",
                                  "one_residue", "no_residue"])
def test_refusals_raise_value_error_before_any_launch(case):
    from esm_b200 import MSATransformer, jacobian
    model = _esm2()
    tokens = _tokens(model)
    if case == "msa":
        args = argparse.Namespace(layers=1, embed_dim=128, ffn_embed_dim=512, attention_heads=2, dropout=0.0,
                                  attention_dropout=0.0, activation_dropout=0.0, max_tokens_per_msa=2 ** 14,
                                  max_tokens=2 ** 14, max_positions=1024, embed_positions_msa=True)
        model = MSATransformer(args, "msa_transformer").eval()
        tokens = tokens[:, None]
    elif case == "fp8":
        model.set_precision("fp8")
    elif case == "batch":
        tokens = tokens.expand(2, -1)
    elif case == "1d":
        tokens = tokens[0]
    elif case == "3d":
        tokens = tokens[None]
    elif case == "float":
        tokens = tokens.float()
    elif case == "padding":
        tokens = torch.cat([tokens, torch.tensor([[model.padding_idx]])], 1)
    elif case == "no_cls":
        tokens = tokens[:, 1:]
    elif case == "no_eos":
        tokens = tokens[:, :-1]
    elif case == "one_residue":
        tokens = _tokens(model, "M")
    elif case == "no_residue":
        tokens = _tokens(model, "")
    with pytest.raises(ValueError):
        jacobian.categorical_jacobian(model, tokens)


def test_esm1b_beyond_its_positions_gets_the_stack_length_error():
    from esm_b200 import jacobian
    model = _esm1b()
    tokens = _tokens(model, "A" * 1023)  # T = 1025 > 1024
    with pytest.raises(ValueError, match="above maximum"):
        jacobian.categorical_jacobian(model, tokens)


def test_contact_kernel_wrapper_refuses_bad_shapes_on_the_host():
    from esm_b200 import _lib, jacobian
    with pytest.raises(_lib.Esmb200Error):
        jacobian.jacobian_contacts(torch.zeros((3, 20, 3, 20)))  # host tensor: no fallback


# ---- the command line -------------------------------------------------------------------------------------------
def test_cli_parser():
    from esm_b200 import jacobian_cli, variants
    p = jacobian_cli.create_parser()
    a = p.parse_args(["esm2_t33_650M_UR50D", "seqs.fasta", "out"])
    assert a.model_location == "esm2_t33_650M_UR50D" and str(a.fasta_file) == "seqs.fasta" and str(a.output_dir) == "out"
    assert a.max_tokens == variants.DEFAULT_MAX_TOKENS and a.precision == "fp16"
    assert not a.cpu_offload and not a.save_jacobian
    a = p.parse_args(["m.pt", "s.fa", "o", "--max-tokens", "4096", "--precision", "fp32x3", "--cpu-offload",
                      "--save-jacobian"])
    assert a.max_tokens == 4096 and a.precision == "fp32x3" and a.cpu_offload and a.save_jacobian
    with pytest.raises(SystemExit):
        p.parse_args(["m.pt", "s.fa", "o", "--precision", "fp8"])
    with pytest.raises(SystemExit):
        p.parse_args(["m.pt", "s.fa"])


def test_cli_refuses_a_random_init_model(tmp_path, monkeypatch):
    from esm_b200 import jacobian_cli
    monkeypatch.setenv("ESMB200_ALLOW_RANDOM_INIT", "1")
    fasta = tmp_path / "s.fa"
    fasta.write_text(">a\nMKTAYIAKQR\n")
    args = jacobian_cli.create_parser().parse_args(["esm2_t6_8M_UR50D", str(fasta), str(tmp_path / "out")])
    with pytest.warns(UserWarning):
        with pytest.raises(RuntimeError, match="random-init"):
            jacobian_cli.run(args)
    assert not (tmp_path / "out").exists()


# ---- the C ABI --------------------------------------------------------------------------------------------------
def test_jacobian_symbols_are_declared_and_exported_at_abi_version_4():
    from esm_b200 import _lib
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "esmb200.h")).read(), flags=re.S)
    for name in ("esmb200_jacobian_scratch_bytes", "esmb200_jacobian_contacts"):
        assert re.search(rf"\b{name}\s*\(", text), name
        assert name in _lib.EXPORTS
    assert re.search(r"#define ESMB200_ABI_VERSION 4\b", text)
    assert _lib.ABI_VERSION == 4
    assert _lib.load().esmb200_abi_version() == 4


@pytest.mark.parametrize("L,nbytes", [(0, 0), (1, 0), (2, 23296), (3, 33280), (17, 169984), (64, 651520),
                                      (1022, 67243008), (3000, 542451456)])
def test_jacobian_scratch_bytes_are_pinned(L, nbytes):
    """fp64 S_i, S_j, S, the 64-wide j-tile partials of S_j, N and its row and column sums, each 256-byte aligned."""
    from esm_b200 import _lib
    assert _lib.load().esmb200_jacobian_scratch_bytes(L) == nbytes
    if L >= 2:
        tiles = (L + 63) // 64
        parts = [400 * L, 400 * L, 400, tiles * L * 400, L * L, L, L]
        assert nbytes == sum((8 * p + 255) // 256 * 256 for p in parts)
