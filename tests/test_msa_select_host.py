"""CPU: greedy row selection for the MSA Transformer (esm_b200.msa_select) without a GPU. The numpy restatement in
tests/msa_select_refs.py against the rows the reference notebook's greedy_select returned (tests/golden/msa_select.json),
the paths that need no launch, the refusals of the Python entry points, the --msa-select flags and the new symbols."""
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # msa_select_refs

import msa_select_refs as ref  # noqa: E402


CASES = ref.fixture_cases()


def test_the_fixture_covers_the_summation_edges():
    assert len(CASES) == 66 and {m for _, _, m, _ in CASES} == {"max", "min"}
    ks = {k for msa, k, _, _ in CASES if len(msa) > k}
    assert any(8 < k <= 128 for k in ks) and any(128 < k <= 256 for k in ks) and any(k > 256 for k in ks)
    assert {len(msa[0][1]) for msa, _, _, _ in CASES} >= {1, 3, 7, 10}
    assert {0, 1} <= {k for _, k, _, _ in CASES} and any(len(msa) == 1 for msa, _, _, _ in CASES)


@pytest.mark.parametrize("i", range(len(CASES)))
def test_the_restatement_picks_the_notebook_rows(i):
    msa, k, mode, selected = CASES[i]
    order = ref.greedy_order(ref.as_rows(msa), k, mode)
    if len(msa) > k:
        assert order[0] == 0 and len(order) == max(k, 1) and len(set(order)) == len(order)
    assert sorted(order) == selected


@pytest.mark.parametrize("mode", ["max", "min"])
def test_the_loop_without_the_shortcut_runs_to_k_equal_n(mode):
    """shortcut=False at k = N picks every row once, starting at the query, and its first k' picks are the picks at
    k' < N: the last step, with one candidate left, takes it."""
    rows = np.random.default_rng(4).integers(0, 3, (140, 9)).astype(np.uint8)
    order = ref.greedy_order(rows, 140, mode, shortcut=False)
    assert ref.greedy_order(rows, 140, mode) == list(range(140))
    assert order[0] == 0 and sorted(order) == list(range(140))
    for k in (1, 2, 9, 130, 139):
        assert order[:k] == ref.greedy_order(rows, k, mode)
    with pytest.raises(AssertionError):
        ref.greedy_order(rows, 141, mode, shortcut=False)


def test_a_running_sum_is_not_the_rule():
    """On at least one fixture case past 8 picks, a running mean in selection order picks other rows."""
    def running(rows, k, mode):
        sel, acc = [0], np.zeros(len(rows))
        for t in range(1, k):
            acc = acc + (rows != rows[sel[-1]]).sum(1) / rows.shape[1]
            score = acc / t
            score[sel] = -np.inf if mode == "max" else np.inf
            sel.append(int(np.argmax(score) if mode == "max" else np.argmin(score)))
        return sorted(sel)

    assert any(running(ref.as_rows(msa), k, mode) != sel for msa, k, mode, sel in CASES if len(msa) > k > 8)


def test_no_launch_when_every_row_or_only_the_query_is_kept_and_the_refusals():
    from esm_b200 import msa_select
    for msa, k, mode, selected in CASES:
        if len(msa) <= k or k <= 1:
            got = msa_select.greedy_select(msa, k, mode)
            assert got == [msa[i] for i in selected] and (got is msa) == (len(msa) <= k)
    ragged = [("q", "MKV"), ("a", "MK"), ("b", "MKVL")]
    for k in (0, 1, 2):
        with pytest.raises(ValueError, match="same length"):
            msa_select.greedy_select(ragged, k)
        with pytest.raises(ValueError):
            ref.as_rows(ragged)  # the notebook's np.array raises it
    with pytest.raises(ValueError, match="'max' or 'min'"):
        msa_select.greedy_select([("q", "MKV")] * 3, 2, mode="mean")


def test_cli_flags_parse_and_default_to_the_first_rows(tmp_path):
    from esm_b200 import predict_cli, sample_msa_cli, variants
    a = predict_cli.create_parser().parse_args([])
    assert a.msa_select == "first" and a.msa_samples == 400
    assert predict_cli.create_parser().parse_args(["--msa-select", "min"]).msa_select == "min"
    p = sample_msa_cli.create_parser()
    a = p.parse_args(["m.pt", "--msa", "x.a3m", "--out", "d"])
    assert a.msa_select == "first" and a.msa_samples is None
    with pytest.raises(SystemExit):
        p.parse_args(["m.pt", "--msa", "x.a3m", "--msa-select", "hhfilter", "--out", "d"])
    (tmp_path / "in.a3m").write_text(">q\nMKTAYIAKQR\n>h\nMK-AYLAKQR\n>g\nMKtTAYLAKQR\n")
    for n in (2, None):
        assert predict_cli.read_alignment(tmp_path / "in.a3m", n) == variants.read_msa(tmp_path / "in.a3m", n)
    for mode in ("max", "min"):  # refused before the model is loaded
        args = p.parse_args(["missing.pt", "--msa", str(tmp_path / "in.a3m"), "--msa-select", mode, "--out",
                             str(tmp_path / "out")])
        with pytest.raises(ValueError, match="give --msa-samples"):
            sample_msa_cli.run(args)


def test_symbols_are_declared_and_exported():
    from esm_b200 import _lib
    text = open(os.path.join(os.path.dirname(HERE), "include", "esmb200.h")).read()
    lib = _lib.load()
    for name in ("esmb200_msa_select_scratch_bytes", "esmb200_msa_greedy_select"):
        assert re.search(rf"\b{name}\s*\(", text) and name in _lib.EXPORTS and hasattr(lib, name)
    assert re.search(r"#define ESMB200_SELECT_MAX 0\b", text) and _lib.SELECT_MAX == 0
    assert re.search(r"#define ESMB200_SELECT_MIN 1\b", text) and _lib.SELECT_MIN == 1
    # counts uint16 [k - 1, N] | d fp64 [C + 1] | picked [N] | partials fp64 + int32 [ceil(N / 256)] | ticket
    assert lib.esmb200_msa_select_scratch_bytes(10000, 256, 128) == 2540032 + 2304 + 10240 + 512 + 256 + 256
