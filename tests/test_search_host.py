"""CPU: nearest-neighbour search (esm_b200.search) without a GPU. The float64 restatement in tests/search_refs.py
(exact scores, the (score descending, index ascending) order, the ambiguity band and the check the GPU results are
held to), the index's build / save / load round trip, from_extract_dir on synthetic extract_cli files, every Python
refusal, the CLI parsers, the new symbols, and the C-ABI refusals with placeholder pointers."""
import ctypes
import os
import re
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # search_refs, kernel_refs

import search_refs as ref  # noqa: E402


def _rows(n, E, metric, seed):
    from esm_b200 import search
    return search.prepare_rows(torch.randn(n, E, generator=torch.Generator().manual_seed(seed)), metric)


# ---- the restatement -------------------------------------------------------------------------------------------------
def test_exact_scores_and_the_order():
    a, x = _rows(5, 100, "l2", 0), _rows(40, 100, "l2", 1)
    beta = -x.double().pow(2).sum(1)
    s, tol = ref.exact(a, x, 2.0, beta)
    want = 2 * a.double() @ x.double().T + beta[None]
    assert torch.equal(s, want) and bool((tol > 0).all())
    # -|a - x|^2 = s - |a|^2: the order of s is the order of distance
    d = torch.cdist(a.double(), x.double()) ** 2
    assert torch.allclose(-d, s - a.double().pow(2).sum(1, keepdim=True), atol=1e-9)
    ss = torch.tensor([[1.0, 3.0, 3.0, 2.0, 3.0]], dtype=torch.float64)
    top, idx = ref.topk_exact(ss, 4, torch.ones_like(ss, dtype=torch.bool))
    assert idx.tolist() == [[1, 2, 4, 3]] and top.tolist() == [[3.0, 3.0, 3.0, 2.0]]
    mask = ref.candidates_mask(1, 5, 1, "cpu")
    assert ref.topk_exact(ss, 2, mask)[1].tolist() == [[2, 4]]


def test_candidates_mask_leaves_out_i_plus_offset():
    m = ref.candidates_mask(4, 5, 2, "cpu")
    assert (~m).nonzero().tolist() == [[0, 2], [1, 3], [2, 4]]
    m = ref.candidates_mask(2, 5, 0, "cpu", q0=3)
    assert (~m).nonzero().tolist() == [[0, 3], [1, 4]]
    assert bool(ref.candidates_mask(3, 3, -1, "cpu").all())


def test_the_band_is_one_wide_on_random_rows_and_covers_ties():
    a, x = _rows(20, 320, "cosine", 2), _rows(500, 320, "cosine", 3)
    s, tol = ref.exact(a, x)
    mask = torch.ones_like(s, dtype=torch.bool)
    w = ref.band_width(s, tol, 10, mask)
    assert bool((w >= 1).all()) and float(w.float().mean()) < 1.5
    xd = torch.cat([x[:5], x[:5], x[5:]])  # five rows twice
    s, tol = ref.exact(a, xd)
    top, idx = ref.topk_exact(s, 1, torch.ones_like(s, dtype=torch.bool))
    assert bool((w >= 1).all())
    dup = idx[:, 0] < 10
    assert bool((ref.band_width(s, tol, 1, torch.ones_like(s, dtype=torch.bool))[dup] >= 2).all())


def test_check_accepts_the_exact_answer_and_catches_faults():
    a, x = _rows(30, 256, "cosine", 4), _rows(600, 256, "cosine", 5)
    s, tol = ref.exact(a, x)
    mask = torch.ones_like(s, dtype=torch.bool)
    top, idx = ref.topk_exact(s, 10, mask)
    scores = top.float()
    ref.check(scores, idx, s, tol, mask)
    bad = idx.clone()
    bad[:, 9] = torch.sort(-s, dim=1, stable=True).indices[:, 300]  # a candidate far below the band
    with pytest.raises(AssertionError, match="ambiguity band"):
        ref.check(s.gather(1, bad).float(), bad, s, tol, mask)
    with pytest.raises(AssertionError, match="past the bound"):
        ref.check(scores + 1e-3, idx, s, tol, mask)
    with pytest.raises(AssertionError, match="ordered"):
        ref.check(scores.flip(1), idx.flip(1), s, tol, mask)
    with pytest.raises(AssertionError, match="twice"):
        ref.check(scores, torch.cat([idx[:, :1], idx[:, :9]], 1), s, tol, mask)
    with pytest.raises(AssertionError, match="left-out"):
        ref.check(scores, idx, s, tol, mask.scatter(1, idx[:, :1], False))


# ---- the index -------------------------------------------------------------------------------------------------------
def test_rows_are_normalised_padded_and_rounded():
    from esm_b200 import search
    x = torch.randn(7, 480, generator=torch.Generator().manual_seed(6)) * 3
    rows = search.prepare_rows(x, "cosine")
    assert rows.shape == (7, 512) and rows.dtype == torch.float16 and bool((rows[:, 480:] == 0).all())
    want = (x.double() / x.double().norm(dim=1, keepdim=True)).half()
    assert torch.equal(rows[:, :480], want)
    rows = search.prepare_rows(x, "l2")
    assert torch.equal(rows[:, :480], x.double().half())
    assert torch.equal(search.squared_norms(rows), rows.double().pow(2).sum(1).float())
    assert search.padded_dim(320) == 320 and search.padded_dim(1) == 64 and search.padded_dim(5120) == 5120


def test_splits_fill_the_gpu_about_twice():
    from esm_b200 import search
    assert search.choose_splits(1, 570_000, 132) == 264
    assert search.choose_splits(1024, 570_000, 132) == 17
    assert search.choose_splits(100_000, 100_000, 132) == 1
    assert search.choose_splits(1, 300, 132) == 2
    assert search.choose_splits(1, 10**9, 1000) == 1024


def test_save_load_round_trip(tmp_path):
    from esm_b200 import search
    x = torch.randn(33, 100, generator=torch.Generator().manual_seed(7))
    for metric in ("cosine", "l2"):
        index = search.EmbeddingIndex(x, [f"p{i}" for i in range(33)], metric, layer=6)
        index.save(tmp_path / "db.pt")
        back = search.EmbeddingIndex.load(tmp_path / "db.pt", device="cpu")
        assert torch.equal(back.rows, index.rows) and back.labels == index.labels and back.metric == metric
        assert back.layer == 6 and back.dim == 100 and len(back) == 33
        if metric == "l2":
            assert torch.equal(back.sqnorm, index.sqnorm)
    torch.save({"rows": x}, tmp_path / "other.pt")
    with pytest.raises(ValueError, match="not a saved EmbeddingIndex"):
        search.EmbeddingIndex.load(tmp_path / "other.pt", device="cpu")


def _write(root, label, vec, layer):
    path = root / f"{label}.pt"
    path.parent.mkdir(parents=True, exist_ok=True)
    torch.save({"label": label, "representations": {layer: vec[None].repeat(3, 1)},
                "mean_representations": {layer: vec.clone()}}, path)


def test_from_extract_dir_reads_nested_labels_in_label_order(tmp_path):
    from esm_b200 import search
    g = torch.Generator().manual_seed(8)
    labels = ["zeta", "sp|P1|A/b", "alpha", "sp|P1|A/a", "m/n/o"]
    vecs = {l: torch.randn(320, generator=g) for l in labels}
    for l in labels:
        _write(tmp_path, l, vecs[l], 33)
    index = search.EmbeddingIndex.from_extract_dir(tmp_path, layer=33, metric="l2")
    assert index.labels == sorted(labels) and index.layer == 33 and index.dim == 320
    want = torch.stack([vecs[l] for l in sorted(labels)]).half()
    assert torch.equal(index.rows, want)


def test_from_extract_dir_refusals(tmp_path):
    from esm_b200 import search
    g = torch.Generator().manual_seed(9)
    _write(tmp_path / "a", "p1", torch.randn(320, generator=g), 33)
    _write(tmp_path / "a", "p2", torch.randn(320, generator=g), 12)
    with pytest.raises(ValueError, match=r"p2\.pt has no mean_representations\[33\]"):
        search.EmbeddingIndex.from_extract_dir(tmp_path / "a", layer=33)
    _write(tmp_path / "b", "p1", torch.randn(320, generator=g), 33)
    _write(tmp_path / "b", "sub/p2", torch.randn(480, generator=g), 33)
    with pytest.raises(ValueError, match="width 480"):
        search.EmbeddingIndex.from_extract_dir(tmp_path / "b", layer=33)
    (tmp_path / "c").mkdir()
    with pytest.raises(ValueError, match="no .pt files"):
        search.EmbeddingIndex.from_extract_dir(tmp_path / "c", layer=33)
    with pytest.raises(ValueError, match="metric"):
        search.EmbeddingIndex.from_extract_dir(tmp_path / "b", layer=33, metric="dot")


def test_python_refusals_on_a_cpu_index():
    from esm_b200 import search
    x = torch.randn(20, 64, generator=torch.Generator().manual_seed(10))
    with pytest.raises(ValueError, match="metric"):
        search.EmbeddingIndex(x, metric="cos")
    with pytest.raises(ValueError, match="non-finite"):
        search.EmbeddingIndex(torch.cat([x, torch.full((1, 64), float("inf"))]))
    with pytest.raises(ValueError, match="zero row"):
        search.EmbeddingIndex(torch.cat([x, torch.zeros(1, 64)]))
    with pytest.raises(ValueError, match="fp16 range"):
        search.EmbeddingIndex(x * 1e5, metric="l2")
    search.EmbeddingIndex(x * 1e5, metric="cosine")  # normalised before rounding: fine
    with pytest.raises(ValueError, match="labels"):
        search.EmbeddingIndex(x, labels=["a"])
    with pytest.raises(TypeError):
        search.EmbeddingIndex(x.numpy())
    with pytest.raises(TypeError):
        search.EmbeddingIndex(torch.ones(20, 64, dtype=torch.int64))
    with pytest.raises(ValueError, match="at least one row"):
        search.EmbeddingIndex(torch.zeros(0, 64))
    index = search.EmbeddingIndex(x, metric="cosine")
    for k in (0, 21, 129):
        with pytest.raises(ValueError, match=r"k must be in \[1, 20\]"):
            index.search(x[:2], k=k)
    with pytest.raises(TypeError):
        index.search(x[:2], k=2.0)
    with pytest.raises(ValueError, match=r"k must be in \[1, 19\]"):
        index.search_all(k=20)
    with pytest.raises(ValueError, match="width 65"):
        index.search(torch.randn(2, 65), k=3)
    with pytest.raises(ValueError, match="non-finite"):
        index.search(torch.full((2, 64), float("nan")), k=3)
    with pytest.raises(ValueError, match="zero row"):
        index.search(torch.zeros(2, 64), k=3)
    with pytest.raises(ValueError, match="fp16 range"):
        search.EmbeddingIndex(x, metric="l2").search(x[:2] * 1e5, k=3)
    with pytest.raises(ValueError, match="on the CPU"):
        index.search(x[:2], k=3)
    with pytest.raises(ValueError, match="on the CPU"):
        index.search_all(k=3)


# ---- the command line ------------------------------------------------------------------------------------------------
def test_cli_parsers():
    from esm_b200 import search_cli
    p = search_cli.create_parser()
    a = p.parse_args(["build", "ex", "--layer", "33", "--out", "db.pt"])
    assert a.command == "build" and a.layer == 33 and a.metric == "cosine" and str(a.out) == "db.pt"
    assert p.parse_args(["build", "ex", "--layer", "6", "--metric", "l2", "--out", "d"]).metric == "l2"
    a = p.parse_args(["query", "db.pt", "--queries", "qdir", "--k", "5", "--out", "h.tsv"])
    assert a.command == "query" and str(a.queries) == "qdir" and not a.all and a.k == 5
    a = p.parse_args(["query", "db.pt", "--all", "--out", "h.tsv"])
    assert a.all and a.queries is None and a.k == 10
    for bad in (["query", "db.pt", "--out", "h"], ["query", "db.pt", "--all", "--queries", "q", "--out", "h"],
                ["build", "ex", "--out", "d"], ["build", "ex", "--layer", "3", "--metric", "dot", "--out", "d"], []):
        with pytest.raises(SystemExit):
            p.parse_args(bad)


def test_cli_query_refuses_mismatched_queries_before_any_work(tmp_path):
    from esm_b200 import search, search_cli
    g = torch.Generator().manual_seed(12)
    search.EmbeddingIndex(torch.randn(10, 320, generator=g), metric="cosine", layer=33).save(tmp_path / "db.pt")
    _write(tmp_path / "q1", "x", torch.randn(480, generator=g), 33)
    _write(tmp_path / "q2", "x", torch.randn(320, generator=g), 12)
    p = search_cli.create_parser()
    with pytest.raises(ValueError, match="width 480"):
        search_cli.run(p.parse_args(["query", str(tmp_path / "db.pt"), "--queries", str(tmp_path / "q1"),
                                     "--out", str(tmp_path / "h.tsv")]))
    with pytest.raises(ValueError, match=r"mean_representations\[33\]"):
        search_cli.run(p.parse_args(["query", str(tmp_path / "db.pt"), "--queries", str(tmp_path / "q2"),
                                     "--out", str(tmp_path / "h.tsv")]))
    with pytest.raises(ValueError, match=r"k must be in \[1, 9\]"):
        search_cli.run(p.parse_args(["query", str(tmp_path / "db.pt"), "--all", "--k", "10",
                                     "--out", str(tmp_path / "h.tsv")]))
    assert not (tmp_path / "h.tsv").exists()


# ---- the C ABI -------------------------------------------------------------------------------------------------------
def test_symbols_are_declared_and_exported():
    from esm_b200 import _lib
    text = open(os.path.join(os.path.dirname(HERE), "include", "esmb200.h")).read()
    lib = _lib.load()
    for name in ("esmb200_knn_scratch_bytes", "esmb200_knn_search"):
        assert re.search(rf"\b{name}\s*\(", text) and name in _lib.EXPORTS and hasattr(lib, name)
    assert lib.esmb200_abi_version() == 4
    n = ctypes.c_size_t(0)
    assert lib.esmb200_knn_scratch_bytes(1000, 10, 3, ctypes.byref(n)) == 0 and n.value == 1000 * 10 * 3 * 8
    for args in ((1000, 0, 3), (1000, 129, 3), (1000, 10, 0), (1000, 10, 1025), (-1, 10, 3)):
        assert lib.esmb200_knn_scratch_bytes(*args, ctypes.byref(n)) == -1
    assert lib.esmb200_knn_scratch_bytes(10, 10, 3, None) == -1


# The calls pass placeholder pointers, which a refused call never dereferences.  They run only where no CUDA device is
# present, so that a refusal lost from the library can never turn into a kernel launch on a bad address; on a machine
# with a device, tests/test_gpu_search.py repeats every refusal with real buffers.
_FAKE = 4096
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="placeholder pointers: only where nothing can launch")
_ARGS = dict(queries=_FAKE, q_ld=320, Q=8, base=_FAKE, b_ld=320, N=300, D=320, beta=None, alpha=1.0, self_offset=-1,
             k=10, splits=2, scratch=_FAKE, scratch_bytes=1 << 20, out_scores=_FAKE, out_idx=_FAKE)
REFUSALS = [
    ({"queries": None}, "null"), ({"base": None}, "null"), ({"scratch": None}, "null"),
    ({"out_scores": None}, "null"), ({"out_idx": None}, "null"),
    ({"k": 0}, "1 <= k <= 128"), ({"k": 129}, "1 <= k <= 128"),
    ({"N": 5, "k": 6}, "candidates"), ({"self_offset": 0, "N": 10, "k": 10}, "candidates"),
    ({"D": 100}, "D % 64"), ({"D": 0}, "D % 64"),
    ({"q_ld": 300}, "q_ld"), ({"b_ld": 324}, "b_ld"),
    ({"queries": _FAKE + 8}, "16-byte aligned"), ({"base": _FAKE + 2}, "16-byte aligned"),
    ({"splits": 0}, "splits"), ({"splits": 1025}, "splits"),
    ({"scratch_bytes": 8 * 2 * 10 * 8 - 1}, "scratch smaller"),
    ({"Q": -1}, "Q >= 0"), ({"N": 0}, "N < 2^31"), ({"N": 1 << 31}, "N < 2^31"),
]


@no_device
@pytest.mark.parametrize("over,msg", REFUSALS, ids=lambda v: v if isinstance(v, str) else "-".join(v) if isinstance(v, dict) else "")
def test_knn_search_refuses_bad_arguments(over, msg):
    from esm_b200 import _lib
    lib = _lib.load()
    kw = dict(_ARGS, **over)
    before = lib.esmb200_launch_count()
    rc = lib.esmb200_knn_search(*kw.values(), None)
    assert rc == -1 and msg in lib.esmb200_last_error().decode(), lib.esmb200_last_error()
    assert lib.esmb200_launch_count() == before
