"""CPU: the overlapping-window plan of esm_b200.windows (starts, coverage, weights, window tokens), the refusals that
come before any launch, the --window flag of both command lines, and the merge entry point in the C ABI."""
import argparse
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("n,W,want", [
    (2000, 1022, [0, 489, 978]),
    (1022, 1022, [0]),
    (5, 1022, [0]),
    (1023, 1022, [0, 1]),
    (150, 62, [0, 29, 58, 88]),
    (3000, 1022, [0, 494, 989, 1483, 1978]),
    (7, 2, [0, 1, 2, 3, 4, 5]),
])
def test_starts_are_pinned(n, W, want):
    from esm_b200 import windows
    assert windows.starts(n, W) == want


@pytest.mark.parametrize("n,W", [(1, 2), (3, 2), (100, 3), (150, 62), (1025, 1022), (2000, 1022), (2500, 1022),
                                 (34350, 1022), (999, 100), (64, 64), (65, 64)])
def test_every_residue_covered_with_normalised_weights(n, W):
    from esm_b200 import windows
    s = windows.starts(n, W)
    K = len(s)
    if n <= W:
        assert s == [0]
    else:
        assert K == -(-(n - W) // (W // 2)) + 1
        assert s[0] == 0 and s[-1] + W == n
        assert all(0 < b - a <= W // 2 for a, b in zip(s, s[1:]))
    plan = windows.Plan(n, W, 1, 1)
    res, win, off, w = plan.residue_terms()
    assert torch.equal(torch.bincount(res, minlength=n) > 0, torch.ones(n, dtype=torch.bool))
    assert bool((off >= 0).all()) and bool((off < min(n, W)).all())
    assert torch.equal(res, torch.sort(res, stable=True).values)           # residue-major
    sums = torch.zeros(n, dtype=torch.float64).index_add_(0, res, w.double())
    assert float((sums - 1).abs().max()) <= 1e-6
    single = torch.bincount(res, minlength=n)[res] == 1
    assert bool((w[single] == 1.0).all())                                    # exactly 1.0 with one window
    # the taper: min(o + 1, W - o), normalised over the covering windows
    for p in {0, n // 3, n // 2, n - 1}:
        sel = res == p
        taper = torch.minimum(off[sel] + 1, W - off[sel]).double()
        assert torch.allclose(w[sel].double(), taper / taper.sum(), rtol=1e-6, atol=0)
        assert torch.equal(win[sel], torch.sort(win[sel]).values)           # window order


def test_terms_take_cls_from_the_first_window_and_eos_from_the_last():
    from esm_b200 import windows
    plan = windows.Plan(150, 62, 1, 1)
    pos, win, row, w = plan.terms()
    assert torch.equal(pos, torch.sort(pos, stable=True).values)
    assert (pos[0].item(), win[0].item(), row[0].item(), w[0].item()) == (0, 0, 0, 1.0)
    assert (pos[-1].item(), win[-1].item(), row[-1].item(), w[-1].item()) == (151, 3, 63, 1.0)
    assert set(torch.bincount(pos).tolist()) <= {1, 2, 3}


def test_window_tokens_are_the_tokenised_crops():
    from esm_b200 import Alphabet, windows
    alphabet = Alphabet.from_architecture("ESM-1b")
    g = torch.Generator().manual_seed(0)
    seq = "".join("LAGVSERTIDPKQNFYMHWC"[i] for i in torch.randint(0, 20, (150,), generator=g).tolist())
    _, _, full = alphabet.get_batch_converter()([("p", seq)])
    plan = windows.Plan(150, 62, 1, 1)
    _, _, crops = alphabet.get_batch_converter()([(str(k), seq[s:s + 62]) for k, s in enumerate(plan.starts)])
    ext = torch.cat([full[0], torch.tensor([alphabet.padding_idx])])
    assert torch.equal(ext[plan.gather(full.shape[1], 64)], crops)
    # a wider batch pads each window on the right
    g70 = ext[plan.gather(full.shape[1], 70)]
    assert torch.equal(g70[:, :64], crops) and bool((g70[:, 64:] == alphabet.padding_idx).all())


def _esm1b(max_positions=64):
    from esm_b200 import ProteinBertModel
    args = argparse.Namespace(arch="roberta_large", layers=1, embed_dim=64, ffn_embed_dim=256, attention_heads=2,
                              max_positions=max_positions, emb_layer_norm_before=True, token_dropout=True)
    return ProteinBertModel(args, "ESM-1b")


def test_refusals_before_any_launch():
    from esm_b200 import ESM2, variants, windows
    esm1b = _esm1b(64)
    esm2 = ESM2(num_layers=1, embed_dim=64, attention_heads=2)
    assert windows.check_window(esm1b, 62) == 62
    assert windows.check_window(esm2, 5000) == 5000
    for model in (esm1b, esm2):
        for bad in (1, 0, -3):
            with pytest.raises(ValueError, match="at least 2"):
                windows.check_window(model, bad)
    with pytest.raises(TypeError):
        windows.check_window(esm2, 2.5)
    with pytest.raises(ValueError, match="learned positions"):
        windows.check_window(esm1b, 63)                                      # 63 + 2 > 64
    tokens = torch.zeros((1, 200), dtype=torch.int64)
    # the models sit on the CPU: a launch would raise Esmb200Error, so a ValueError shows the check came first
    with pytest.raises(ValueError):
        esm1b.forward_windowed(tokens, 63)
    with pytest.raises(ValueError):
        esm2.forward_windowed(tokens, 1)
    with pytest.raises(ValueError):
        variants.masked_marginals(esm1b, tokens, window=63)
    with pytest.raises(ValueError):
        variants.wt_marginals(esm1b, tokens, window=1)
    with pytest.raises(ValueError):
        variants.pseudo_ppl(esm1b, esm1b.alphabet, "ACDE" * 50, ["A1C"], window=63)


def test_predict_cli_window_flag(tmp_path):
    from esm_b200 import predict_cli
    base = ["--model-location", "m.pt", "--sequence", "ACD", "--dms-input", "in.csv", "--dms-output", "out.csv"]
    assert predict_cli.create_parser().parse_args(base).window is None
    assert predict_cli.create_parser().parse_args(base + ["--window", "1022"]).window == 1022
    with pytest.raises(SystemExit):
        predict_cli.create_parser().parse_args(base + ["--window", "x"])
    # an MSA model location is refused before the table is read or any model is loaded
    args = predict_cli.create_parser().parse_args(
        ["--model-location", "esm_msa1b_t12_100M_UR50S", "--sequence", "ACD", "--dms-input",
         str(tmp_path / "missing.csv"), "--dms-output", str(tmp_path / "out.csv"), "--scoring-strategy",
         "masked-marginals", "--window", "100"])
    with pytest.raises(ValueError, match="not windowed"):
        predict_cli.run(args)
    args.window = 1
    with pytest.raises(ValueError, match="at least 2"):
        predict_cli.run(args)
    assert not (tmp_path / "out.csv").exists()


def test_extract_cli_window_flag(tmp_path):
    from esm_b200 import extract_cli
    base = ["esm1v_t33_650M_UR90S_1", str(tmp_path / "in.fasta"), str(tmp_path / "out")]
    args = extract_cli.create_parser().parse_args(base + ["--include", "mean"])
    assert args.window is None
    args = extract_cli.create_parser().parse_args(base + ["--include", "mean", "per_tok", "--window", "1022"])
    assert args.window == 1022
    # --window with contacts is refused before any work (no device, no model, no output directory)
    args = extract_cli.create_parser().parse_args(base + ["--include", "mean", "contacts", "--window", "1022"])
    with pytest.raises(ValueError, match="contacts"):
        extract_cli.run(args)
    assert not (tmp_path / "out").exists()


def test_merge_entry_point_is_exported_at_abi_version_4():
    from esm_b200 import _lib
    header = open(os.path.join(ROOT, "include", "esmb200.h")).read()
    assert re.search(r"\bint esmb200_window_merge\(", header)
    assert "esmb200_window_merge" in _lib.EXPORTS
    assert re.search(r"#define ESMB200_ABI_VERSION 4\b", header)
    assert _lib.ABI_VERSION == 4
