"""CPU: the host side of variant-effect scoring (esm_b200.variants, esm_b200.predict_cli) against the reference's
examples/variant-prediction/predict.py: mutation parsing and label_row's arithmetic, read_msa, the command line, the
output table and the model routing. The scores themselves are checked on the GPU (tests/test_gpu_variants.py)."""
import csv
import io
import json
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # variant_fixtures (tests/variant_fixtures.py)


@pytest.fixture(scope="module")
def fixture(golden_dir):
    with open(os.path.join(golden_dir, "variants.json")) as f:
        return json.load(f)


def test_parse_mutation_and_offset():
    from esm_b200.variants import parse_mutation
    assert parse_mutation("A1B") == ("A", 1, "B")
    assert parse_mutation("A1B", offset_idx=1) == ("A", 0, "B")
    assert parse_mutation("W263X", offset_idx=24) == ("W", 239, "X")


def test_label_scores_is_label_row():
    """predict.py:107-115: lp[1 + idx, mt] - lp[1 + idx, wt] in fp32; letters outside the alphabet are <unk>."""
    from esm_b200 import Alphabet
    from esm_b200.variants import label_scores
    a = Alphabet.from_architecture("ESM-1b")
    seq = "MKTAYIAK"
    g = torch.Generator().manual_seed(0)
    lp = torch.randn(1, len(seq) + 2, len(a), generator=g) * 5
    got = label_scores(lp, a, seq, ["M1A", "K8X", "T3J"], offset_idx=1)
    want = [(lp[0, 1, a.get_idx("A")] - lp[0, 1, a.get_idx("M")]).item(),
            (lp[0, 8, a.get_idx("X")] - lp[0, 8, a.get_idx("K")]).item(),
            (lp[0, 3, a.unk_idx] - lp[0, 3, a.get_idx("T")]).item()]
    assert got == want
    assert all(type(v) is float for v in got)
    assert label_scores(lp[0], a, seq, ["M1A"], offset_idx=1) == got[:1]  # [T, V] accepted as well


def test_wild_type_mismatch_raises_the_reference_assertion():
    from esm_b200 import Alphabet
    from esm_b200.variants import label_scores, pseudo_ppl
    a = Alphabet.from_architecture("ESM-1b")
    lp = torch.zeros(1, 6, len(a))
    with pytest.raises(AssertionError, match="The listed wildtype does not match the provided sequence"):
        label_scores(lp, a, "MKTA", ["K1A"], offset_idx=1)
    with pytest.raises(AssertionError, match="The listed wildtype does not match the provided sequence"):
        pseudo_ppl(None, a, "MKTA", ["M2A"], offset_idx=0)  # checked before anything runs


def test_read_msa_removes_insertions_and_keeps_descriptions(tmp_path):
    from esm_b200.variants import read_msa, remove_insertions
    assert remove_insertions("AB-cd.E*f") == "AB-E"
    p = tmp_path / "x.a3m"
    p.write_text("ignored line\n>q the query  \nMKT-A\nYI\n>hit1 score=3 desc\nMKkt.T-A\nY*I\n>hit2\nMK..T-AYI\n")
    assert read_msa(p, 400) == [("q the query", "MKT-AYI"), ("hit1 score=3 desc", "MKT-AYI"), ("hit2", "MKT-AYI")]
    assert read_msa(p, 2) == [("q the query", "MKT-AYI"), ("hit1 score=3 desc", "MKT-AYI")]


def test_read_msa_on_the_fixture_alignment(fixture, tmp_path):
    from esm_b200.variants import read_msa
    p = tmp_path / "msa.a3m"
    p.write_text(fixture["a3m"])
    msa = read_msa(p, fixture["msa_samples"])
    assert len(msa) == fixture["msa_samples"]
    assert msa[0] == ("query 52 residues", fixture["sequence"])
    assert all(len(s) == len(fixture["sequence"]) for _, s in msa)
    assert all(d.endswith("desc with spaces") for d, _ in msa[1:])


def test_cli_flags_and_defaults_match_predict_py():
    """predict.py:45-104, plus --max-tokens."""
    from esm_b200 import predict_cli, variants
    p = predict_cli.create_parser()
    args = p.parse_args(["--model-location", "a.pt", "b", "--sequence", "MKT", "--dms-input", "in.csv",
                         "--dms-output", "out.csv"])
    assert args.model_location == ["a.pt", "b"]
    assert args.mutation_col == "mutant" and args.offset_idx == 0 and args.scoring_strategy == "wt-marginals"
    assert args.msa_path is None and args.msa_samples == 400 and args.nogpu is False
    assert args.max_tokens == variants.DEFAULT_MAX_TOKENS
    assert str(args.dms_input) == "in.csv" and str(args.dms_output) == "out.csv"
    opts = {a.dest: a for a in p._actions}
    assert opts["scoring_strategy"].choices == ["wt-marginals", "pseudo-ppl", "masked-marginals"]
    assert {"model_location", "sequence", "dms_input", "mutation_col", "dms_output", "offset_idx", "scoring_strategy",
            "msa_path", "msa_samples", "nogpu", "max_tokens"} <= set(opts)
    with pytest.raises(SystemExit):
        p.parse_args(["--scoring-strategy", "entropy"])


def test_nogpu_raises(tmp_path):
    from esm_b200 import predict_cli
    args = predict_cli.create_parser().parse_args(["--model-location", "esm1v_t33_650M_UR90S_1", "--sequence", "MK",
                                                   "--dms-input", str(tmp_path / "missing.csv"),
                                                   "--dms-output", str(tmp_path / "o.csv"), "--nogpu"])
    with pytest.raises(RuntimeError, match="no CPU path"):
        predict_cli.run(args)
    assert not (tmp_path / "o.csv").exists()


def test_output_table_reproduces_predict_py_byte_for_byte(fixture, tmp_path):
    """Index column, the input columns exactly as read (quoted cells included), one column per model location: with
    the scores read back from predict.py's table, write_table gives predict.py's table."""
    from esm_b200 import predict_cli
    p = tmp_path / "dms.csv"
    p.write_text(fixture["dms_csv"])
    header, rows = predict_cli.read_table(p)
    assert header == ["mutant", "note", "replicate"]
    for key, text in fixture["outputs"].items():
        table = list(csv.reader(io.StringIO(text)))
        loc = table[0][-1]
        out = tmp_path / "out.csv"
        predict_cli.write_table(out, header, rows, {loc: [float(r[-1]) for r in table[1:]]})
        assert out.read_text() == text, key
    # two model locations: two columns, in the order given
    out = tmp_path / "two.csv"
    predict_cli.write_table(out, header, rows, {"m1.pt": [0.5] * len(rows), "esm1v_t33_650M_UR90S_1": [-1.25] * len(rows)})
    table = list(csv.reader(io.StringIO(out.read_text())))
    assert table[0] == ["", "mutant", "note", "replicate", "m1.pt", "esm1v_t33_650M_UR90S_1"]
    assert [r[0] for r in table[1:]] == [str(i) for i in range(len(rows))]
    assert [r[1:4] for r in table[1:]] == rows
    assert all(r[4:] == ["0.5", "-1.25"] for r in table[1:])


def test_model_routing_for_names_and_checkpoints(fixture, tmp_path):
    import variant_fixtures as vf
    from esm_b200 import ESM2, MSATransformer, ProteinBertModel, predict_cli
    for name in ("esm_msa1_t12_100M_UR50S", "esm_msa1b_t12_100M_UR50S"):
        assert predict_cli.is_msa_location(name)
    for name in ("esm2_t33_650M_UR50D", "esm1b_t33_650M_UR50S", "esm1v_t33_650M_UR90S_3"):
        assert not predict_cli.is_msa_location(name)
    kinds = {"esm2": ESM2, "esm1b": ProteinBertModel, "msa": MSATransformer}
    for name, cfg in vf.MODELS.items():
        assert abs(vf.checksum(vf.state_dict(cfg)) - fixture["models"][name]["state_dict_checksum"]) <= 1e-6 * \
            fixture["models"][name]["state_dict_checksum"]
        path = vf.write_checkpoint(name, cfg, str(tmp_path))
        model, alphabet, is_msa = predict_cli.load_model(path)
        assert is_msa == (cfg["kind"] == "msa")
        assert type(model) is kinds[cfg["kind"]]
        assert alphabet.append_eos == (cfg["kind"] != "msa")
        sd = vf.state_dict(cfg)
        got = model.state_dict()
        assert all(torch.equal(got[k], v) for k, v in sd.items() if k != "embed_tokens.weight" and k != "lm_head.weight")


def test_cli_refuses_random_init_models(tmp_path, monkeypatch):
    from esm_b200 import predict_cli
    monkeypatch.setenv("ESMB200_ALLOW_RANDOM_INIT", "1")
    dms = tmp_path / "dms.csv"
    dms.write_text("mutant\nM1A\n")
    args = predict_cli.create_parser().parse_args(["--model-location", "esm2_t6_8M_UR50D", "--sequence", "MKT",
                                                   "--dms-input", str(dms), "--dms-output", str(tmp_path / "o.csv")])
    with pytest.warns(UserWarning):
        with pytest.raises(RuntimeError, match="random-init"):
            predict_cli.run(args)


def test_scorers_have_no_cpu_fallback():
    from esm_b200 import ESM2, _lib, variants
    model = ESM2(num_layers=1, embed_dim=128, attention_heads=2).eval()
    tokens = torch.tensor([[0, 5, 6, 7, 2]])
    with pytest.raises(_lib.Esmb200Error):
        variants.masked_marginals(model, tokens)
    with pytest.raises(_lib.Esmb200Error):
        variants.wt_marginals(model, tokens)
    with pytest.raises(_lib.Esmb200Error):
        variants.log_softmax_rows(torch.zeros(2, 33))


def test_log_softmax_entry_point_is_declared():
    from esm_b200 import _lib
    assert "esmb200_log_softmax_rows" in _lib.EXPORTS
    header = open(os.path.join(os.path.dirname(HERE), "include", "esmb200.h")).read()
    assert "int esmb200_log_softmax_rows(const float* logits, int64_t ld, int32_t n, int32_t V, const int64_t* target," \
        in header


def test_masked_marginals_rejects_positions_outside_the_sequence():
    """Checked on the host, before any copy is built: an index outside [0, L) never reaches the device."""
    from esm_b200 import ESM2, MSATransformer, variants
    model = ESM2(num_layers=1, embed_dim=128, attention_heads=2).eval()
    tokens = torch.tensor([[0, 5, 6, 7, 2]])
    for bad in ([5], [-1], [0, 2, 9]):
        with pytest.raises(ValueError, match=r"positions must lie in \[0, 5\)"):
            variants.masked_marginals(model, tokens, positions=bad)
    with pytest.raises(TypeError):
        variants.masked_marginals(model, tokens, positions=[1.5])
    msa = MSATransformer(layers=1, embed_dim=128, ffn_embed_dim=256, attention_heads=2).eval()
    with pytest.raises(ValueError, match=r"positions must lie in \[0, 4\)"):
        variants.masked_marginals(msa, torch.zeros((1, 3, 4), dtype=torch.int64), positions=[4])


def test_read_table_skips_blank_lines(tmp_path):
    """pandas.read_csv (predict.py:149) skips blank lines; so does the command line's reader."""
    from esm_b200 import predict_cli
    p = tmp_path / "dms.csv"
    p.write_text("mutant,note\nM1A,x\n\nK2R,\"a, b\"\n   \n\n")
    header, rows = predict_cli.read_table(p)
    assert header == ["mutant", "note"]
    assert rows == [["M1A", "x"], ["K2R", "a, b"]]
    out = tmp_path / "out.csv"
    predict_cli.write_table(out, header, rows, {"m.pt": [0.25, -1.0]})
    assert out.read_text() == ',mutant,note,m.pt\n0,M1A,x,0.25\n1,K2R,"a, b",-1.0\n'
