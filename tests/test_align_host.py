"""CPU: embedding alignment (esm_b200.align) without a GPU. The float32 restatement (tests/align_refs.py) on hand-made
cases with known alignments and deliberate ties, local and global on 1 x 1, 1 x n and n x 1, the Python refusals,
the Alignment helpers and the a3m writer (read back by variants.read_msa), align_cli's parser, label lookup and
length checks, and the new C-ABI symbols."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # align_refs

import align_refs as ref  # noqa: E402


# ---- the restatement ------------------------------------------------------------------------------------------------
def test_identity_block_aligns_on_the_diagonal():
    S = -np.ones((6, 6), np.float32)
    np.fill_diagonal(S, 2.0)
    assert ref.align(S, "local", 1.0, 0.5) == (np.float32(12.0), (0, 6), (0, 6), "MMMMMM")
    assert ref.align(S, "global", 1.0, 0.5) == (np.float32(12.0), (0, 6), (0, 6), "MMMMMM")


def test_local_finds_the_embedded_match_and_global_pays_the_ends():
    S = -np.ones((3, 8), np.float32)
    S[0, 3], S[1, 4], S[2, 5] = 3, 3, 3
    assert ref.align(S, "local", 2.0, 1.0) == (np.float32(9.0), (0, 3), (3, 6), "MMM")
    score, q, t, ops = ref.align(S, "global", 2.0, 1.0)
    assert ops == "TTTMMMTT" and (q, t) == ((0, 3), (0, 8)) and score == np.float32(9 - (2 + 1 + 1) - (2 + 1))


def test_an_affine_gap_in_the_query():
    S = -np.ones((6, 4), np.float32)
    for i, j in [(0, 0), (1, 1), (4, 2), (5, 3)]:
        S[i, j] = 5.0
    score, q, t, ops = ref.align(S, "local", 1.0, 0.5)
    assert ops == "MMQQMM" and score == np.float32(20 - 1.5) and (q, t) == ((0, 6), (0, 4))
    assert ref.score_of(S, ops, 0, 0, 1.0, 0.5) == 18.5


def test_ties_follow_the_evaluation_order():
    # every cell 0 and o = e = 0: diagonal wins every tie, so global is a diagonal run then straight border moves
    S = np.zeros((3, 5), np.float32)
    assert ref.align(S, "global", 0.0, 0.0)[3] == "TTMMM"
    # local with a zero maximum ends at (0, 0): the empty alignment
    assert ref.align(-np.ones((4, 4), np.float32), "local", 1.0, 1.0) == (np.float32(0.0), (0, 0), (0, 0), "")
    # two equal local maxima: the smallest i wins, then the smallest j
    S = -np.ones((4, 4), np.float32)
    S[1, 2] = S[2, 0] = S[1, 3] = 2.0
    assert ref.align(S, "local", 5.0, 5.0) == (np.float32(2.0), (1, 2), (2, 3), "M")
    # o == e: open is taken before extend, so E and F never record an extension
    H, E, F, D = ref.dp(np.zeros((4, 4), np.float32) - 1, "global", 1.0, 1.0)
    assert not (D & (ref.E_EXT | ref.F_EXT)).any()


@pytest.mark.parametrize("mode", ["local", "global"])
def test_one_by_one_one_by_n_and_n_by_one(mode):
    assert ref.align(np.array([[0.5]]), mode, 1, 0.1) == (np.float32(0.5), (0, 1), (0, 1), "M")
    s = ref.align(np.array([[-0.5]]), mode, 1, 0.1)
    assert s == ((np.float32(0.0), (0, 0), (0, 0), "") if mode == "local" else (np.float32(-0.5), (0, 1), (0, 1), "M"))
    row = np.array([[-1, -1, 3, -1]], np.float32)
    col = row.T.copy()
    if mode == "local":
        assert ref.align(row, mode, 1, 0.1) == (np.float32(3), (0, 1), (2, 3), "M")
        assert ref.align(col, mode, 1, 0.1) == (np.float32(3), (2, 3), (0, 1), "M")
    else:
        assert ref.align(row, mode, 1, 0.1)[1:] == ((0, 1), (0, 4), "TTMT")
        assert ref.align(col, mode, 1, 0.1)[1:] == ((0, 4), (0, 1), "QQMQ")


def test_the_vectorised_programme_equals_a_cell_by_cell_loop():
    rng = np.random.default_rng(0)
    for mode in ("local", "global"):
        for La, Lb in [(1, 7), (7, 1), (9, 13), (20, 16)]:
            S = rng.integers(-2, 3, (La, Lb)).astype(np.float32)
            H, E, F, D = ref.dp(S, mode, 1.0, 1.0)
            o, e = np.float32(1.0), np.float32(1.0)
            for i in range(1, La + 1):
                for j in range(1, Lb + 1):
                    ev = max(H[i, j - 1] - o, E[i, j - 1] - e)
                    fv = max(H[i - 1, j] - o, F[i - 1, j] - e)
                    h = max(H[i - 1, j - 1] + S[i - 1, j - 1], ev, fv, np.float32(0) if mode == "local" else -np.inf)
                    assert (H[i, j], E[i, j], F[i, j]) == (h, ev, fv)
            score, (q0, q1), (t0, t1), ops = ref.align(S, mode, 1.0, 1.0)
            assert ops.count("M") + ops.count("Q") == q1 - q0 and ops.count("M") + ops.count("T") == t1 - t0
            assert ref.score_of(S, ops, q0, t0, 1.0, 1.0) == float(score)


# ---- the Python API --------------------------------------------------------------------------------------------------
def test_alignment_helpers():
    from esm_b200.align import Alignment
    a = Alignment(3.0, (2, 7), (0, 6), "MMQTTMMQ")
    assert a.cigar() == "2M1Q2T2M1Q" and Alignment(0.0, (0, 0), (0, 0), "").cigar() == ""
    assert a.pairs() == [(2, 0), (3, 1), (5, 4), (6, 5)]


def test_a3m_rows_round_trip_through_read_msa(tmp_path):
    from esm_b200 import align, variants
    query = "MKTAYIAKQR"
    hits = [("local", "GGMKTWYIAKQ", align.Alignment(1.0, (0, 8), (2, 10), "MMMMTMMQM")),
            ("global", "AMKTAYIAKQRC", align.Alignment(1.0, (0, 10), (0, 12), "TMMMMMMMMMMT")),
            ("empty", "WWW", align.Alignment(0.0, (0, 0), (0, 0), ""))]
    text = align.to_a3m(query, hits, "q1")
    assert text.splitlines()[3] == "MKTWyIA-K--" and text.splitlines()[5] == "aMKTAYIAKQRc"
    (tmp_path / "x.a3m").write_text(text)
    rows = variants.read_msa(tmp_path / "x.a3m", None)
    assert [r[0] for r in rows] == ["q1", "local", "global", "empty"]
    assert rows[1][1] == "MKTWIA-K--" and rows[2][1] == "MKTAYIAKQR" and rows[3][1] == "-" * 10
    assert all(len(r[1]) == len(query) for r in rows)
    with pytest.raises(ValueError, match="beyond"):
        align.a3m_row(5, "MKT", align.Alignment(1.0, (0, 6), (0, 3), "MMMQQQ"))


def test_python_refusals_before_any_work():
    from esm_b200 import align
    q, t = torch.randn(5, 64), torch.randn(7, 64)
    for kw, exc, msg in [(dict(mode="semi"), ValueError, "mode"), (dict(gap_open=-1.0), ValueError, "gap_open"),
                         (dict(gap_extend=float("nan")), ValueError, "gap_extend"),
                         (dict(gap_open=float("inf")), ValueError, "gap_open"),
                         (dict(max_cells=0), ValueError, "max_cells"), (dict(max_cells=2.5), ValueError, "max_cells"),
                         (dict(zscore=1), TypeError, "zscore")]:
        with pytest.raises(exc, match=msg):
            align.align_pairs([q], [t], **kw)
    with pytest.raises(ValueError, match="1 queries for 2 targets"):
        align.align_pairs([q], [t, t])
    with pytest.raises(ValueError, match="width 64, the target 65"):
        align.align_pairs([q], [torch.randn(7, 65)])
    with pytest.raises(ValueError, match="no residues"):
        align.align_pairs([torch.zeros(0, 64)], [t])
    with pytest.raises(TypeError):
        align.align_pairs([q.long()], [t])
    with pytest.raises(TypeError):
        align.align_matrices([torch.zeros(3)])
    with pytest.raises(ValueError, match="at least 1"):
        align.align_matrices([torch.zeros(0, 3)])
    with pytest.raises(ValueError, match="non-finite"):
        align.align_matrices([torch.tensor([[float("inf")]])])
    with pytest.raises(ValueError, match="more than max_cells"):
        align._chunks([10, 20, 5], 15)
    assert align._chunks([10, 5, 5, 20, 1], 20) == [(0, 3), (3, 4), (4, 5)]
    assert align._chunks([], 10) == []


# ---- the command line ----------------------------------------------------------------------------------------------
def test_cli_parser():
    from esm_b200 import align, align_cli
    p = align_cli.create_parser()
    a = p.parse_args(["h.tsv", "--queries", "q", "--targets", "t", "--layer", "33", "--out", "o.tsv"])
    assert (a.mode, a.gap_open, a.gap_extend, a.no_zscore, a.max_cells) == ("local", align.GAP_OPEN,
                                                                            align.GAP_EXTEND, False, None)
    a = p.parse_args(["h.tsv", "--queries", "q", "--targets", "t", "--layer", "6", "--mode", "global", "--gap-open",
                      "2", "--gap-extend", "0.5", "--no-zscore", "--max-cells", "1000", "--out", "o", "--fasta",
                      "s.fa", "--a3m", "d"])
    assert (a.mode, a.gap_open, a.gap_extend, a.no_zscore, a.max_cells, str(a.a3m)) == ("global", 2.0, 0.5, True,
                                                                                        1000, "d")
    for bad in (["h.tsv", "--queries", "q", "--targets", "t", "--out", "o"],
                ["h.tsv", "--queries", "q", "--targets", "t", "--layer", "3", "--mode", "semi", "--out", "o"], []):
        with pytest.raises(SystemExit):
            p.parse_args(bad)


def _write(root, label, n, E, layer):
    path = root / f"{label}.pt"
    path.parent.mkdir(parents=True, exist_ok=True)
    torch.save({"label": label, "representations": {layer: torch.randn(n, E)}}, path)


def test_cli_reads_only_the_named_labels_and_refuses_bad_inputs(tmp_path, monkeypatch):
    from esm_b200 import align_cli
    (tmp_path / "hits.tsv").write_text("query\trank\ttarget\tscore\nsp|A/1\t1\tb\t0.9\nsp|A/1\t2\tc\t0.8\n")
    _write(tmp_path / "e", "sp|A/1", 5, 64, 6)
    _write(tmp_path / "e", "b", 4, 64, 6)
    _write(tmp_path / "e", "c", 3, 64, 12)
    (tmp_path / "e" / "unrelated.pt").write_text("not a torch file")  # never opened: not named in the hits
    emb = align_cli.load_embeddings(tmp_path / "e", ["sp|A/1", "b", "sp|A/1"], 6)
    assert sorted(emb) == ["b", "sp|A/1"] and emb["sp|A/1"].shape == (5, 64)
    with pytest.raises(ValueError, match=r"c\.pt has no representations\[6\] \(extract_cli --include per_tok"):
        align_cli.load_embeddings(tmp_path / "e", ["c"], 6)
    with pytest.raises(ValueError, match="not found"):
        align_cli.load_embeddings(tmp_path / "e", ["zz"], 6)
    with pytest.raises(ValueError, match="truncated"):
        align_cli.check_lengths(emb, {"sp|A/1": "MKTAYIA", "b": "MKTA"})
    with pytest.raises(ValueError, match="not in the FASTA"):
        align_cli.check_lengths(emb, {"b": "MKTA"})
    align_cli.check_lengths(emb, {"sp|A/1": "MKTAY", "b": "MKTA"})
    assert align_cli.read_hits(tmp_path / "hits.tsv")[1] == ("sp|A/1", 2, "c", "0.8")
    (tmp_path / "bad.tsv").write_text("a\tb\n")
    with pytest.raises(ValueError, match="not search_cli query output"):
        align_cli.read_hits(tmp_path / "bad.tsv")
    p = align_cli.create_parser()
    base = [str(tmp_path / "hits.tsv"), "--queries", str(tmp_path / "e"), "--targets", str(tmp_path / "e"),
            "--layer", "6", "--out", str(tmp_path / "o.tsv")]
    with pytest.raises(ValueError, match="--a3m needs --fasta"):
        align_cli.run(p.parse_args(base + ["--a3m", str(tmp_path / "a")]))
    (tmp_path / "s.fa").write_text(">sp|A/1\nMKTAYIA\n>b\nMKTA\n>c\nMKT\n")
    _write(tmp_path / "e", "c", 3, 64, 6)
    with pytest.raises(ValueError, match="truncated"):
        align_cli.run(p.parse_args(base + ["--fasta", str(tmp_path / "s.fa")]))
    assert not (tmp_path / "o.tsv").exists()


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def test_symbols_are_declared_and_exported():
    from esm_b200 import _lib
    text = open(os.path.join(os.path.dirname(HERE), "include", "esmb200.h")).read()
    lib = _lib.load()
    for name in ("esmb200_align_scratch_bytes", "esmb200_align_similarity", "esmb200_align"):
        assert re.search(rf"\b{name}\s*\(", text) and name in _lib.EXPORTS and hasattr(lib, name)
    assert re.search(r"23 embedding alignment", text)
    assert lib.esmb200_abi_version() == 4
    # one byte per cell plus 32 per row and column and 1024 per pair, then 16 per target row and pair, 8 per row
    n = lib.esmb200_align_scratch_bytes(3, 100, 200, 6000)
    dir_bytes = 6000 + 32 * 300 + 1024 * 3 + 32
    border = -(-dir_bytes // 256) * 256
    assert n == border + -(-(16 * 203) // 256) * 256 + 8 * 300
    assert lib.esmb200_align_scratch_bytes(-1, 1, 1, 1) == 0


_FAKE = 4096
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="placeholder pointers: only where nothing can launch")


@no_device
def test_align_refusals_with_placeholder_pointers():
    from esm_b200 import _lib
    lib = _lib.load()
    need = lib.esmb200_align_scratch_bytes(2, 10, 14, 70)
    args = [_FAKE, _FAKE, _FAKE, _FAKE, 2, 10, 14, 70, 0, 1.0, 0.1, _FAKE, need, _FAKE, _FAKE, _FAKE, _FAKE, None]
    before = lib.esmb200_launch_count()
    for k, v, msg in [(8, 5, "mode"), (9, -0.5, "penalties"), (10, float("inf"), "penalties"), (4, -1, "P >= 0"),
                      (5, 1, "n_q"), (12, need - 1, "more cells than the scratch"), (0, None, "null"),
                      (11, _FAKE + 16, "256-byte")]:
        a = list(args)
        a[k] = v
        assert lib.esmb200_align(*a) == -1 and msg in lib.esmb200_last_error().decode()
    sim = [_FAKE, _FAKE, 128, _FAKE, _FAKE, _FAKE, 2, 10, 14, 70, 1, _FAKE, _FAKE, need, None]
    for k, v, msg in [(2, 96, "D % 64"), (10, 3, "zscore"), (13, 0, "more cells"), (0, _FAKE + 2, "16-byte")]:
        a = list(sim)
        a[k] = v
        assert lib.esmb200_align_similarity(*a) == -1 and msg in lib.esmb200_last_error().decode()
    assert lib.esmb200_launch_count() == before
    assert lib.esmb200_align(*(args[:4] + [0, 0, 0, 0] + args[8:])) == 0 and lib.esmb200_launch_count() == before
