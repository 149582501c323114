"""GPU: exact k-nearest-neighbour search (esm_b200.search, esmb200_knn_search).

  1. the kernel against the float64 restatement (tests/search_refs.py) on its own fp16 operands, for cosine and l2:
     Q in {1, 63, 64, 65, 1000}, N in {k, 255, 256, 257, ~10^5}, D in {320, 480 -> 512, 1280, 5120}, k in
     {1, 10, 64, 128}: every score within its bound, the order (score descending, index ascending), and the indices
     of the exact top k outside the ambiguity band;
  2. adversarial databases: all-negative cosine scores with N % 256 != 0 (a zero-filled row would win), ascending and
     descending score order (every tile raises the threshold; the queues overflow), blocks of duplicated rows (ties to
     the smaller index), self_offset;
  3. bit-identical outputs across splits, query batching and query order;
  4. every C-ABI refusal with real buffers, launching nothing;
  5. search_cli build / query against the Python API.
"""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # search_refs, kernel_refs

import search_refs as ref  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _operands(Q, N, E, metric, seed):
    g = torch.Generator().manual_seed(seed)
    from esm_b200 import search
    a = search.prepare_rows(torch.randn(Q, E, generator=g), metric).to(DEV)
    x = search.prepare_rows(torch.randn(N, E, generator=g), metric).to(DEV)
    return a, x


def _run(a, x, k, metric, self_offset=-1, splits=None):
    from esm_b200 import search
    beta = -search.squared_norms(x) if metric == "l2" else None
    alpha = 2.0 if metric == "l2" else 1.0
    s, i = search.knn(a, x, k, beta, alpha, self_offset, splits)
    return s, i, alpha, beta


# ---- 1. shapes -----------------------------------------------------------------------------------------------------
SHAPES = [  # Q, N, E, k
    (1, 10, 320, 10),
    (63, 255, 480, 10),
    (64, 256, 1280, 64),
    (65, 257, 320, 128),
    (1000, 257, 480, 1),
    (64, 128, 5120, 128),
    (65, 100_003, 1280, 10),
    (1000, 100_003, 320, 64),
    (1, 100_003, 5120, 128),
    (63, 2049, 1280, 1),
]


@pytest.mark.parametrize("metric", ["cosine", "l2"])
@pytest.mark.parametrize("Q,N,E,k", SHAPES)
def test_the_kernel_matches_the_float64_restatement(Q, N, E, k, metric):
    a, x = _operands(Q, N, E, metric, seed=Q * 7 + N + E + k)
    s, i, alpha, beta = _run(a, x, k, metric)
    assert s.shape == (Q, k) and i.dtype == torch.int64 and s.is_cuda
    ref.check_chunked(s, i, a, x, alpha, beta)


# ---- 2. adversarial databases ----------------------------------------------------------------------------------------
def test_zero_filled_rows_never_win_against_negative_scores():
    """Every cosine score is negative and N % 256 != 0: an unmasked zero-filled row would score 0 and win."""
    from esm_b200 import search
    g = torch.Generator().manual_seed(11)
    q = torch.rand(65, 256, generator=g) + 0.1
    x = -(torch.rand(1000, 256, generator=g) + 0.1)
    a, xr = search.prepare_rows(q, "cosine").to(DEV), search.prepare_rows(x, "cosine").to(DEV)
    s, i, alpha, beta = _run(a, xr, 128, "cosine")
    assert bool((s < 0).all()) and int(i.max()) < 1000
    ref.check_chunked(s, i, a, xr, alpha, beta)


@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("k", [1, 37, 128])
def test_sorted_databases(descending, k):
    """The database ordered by one query's score: ascending, every tile raises every threshold and overflows the
    queues; descending, the first tile holds the answer."""
    a, x = _operands(64, 20_000, 512, "cosine", seed=5 + k)
    order = torch.argsort((a[:1].double() @ x.double().T)[0], descending=descending)
    x = x[order].contiguous()
    s, i, alpha, beta = _run(a, x, k, "cosine", splits=1)
    ref.check_chunked(s, i, a, x, alpha, beta)
    s2, i2, _, _ = _run(a, x, k, "cosine", splits=5)
    assert torch.equal(s, s2) and torch.equal(i, i2)


@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_duplicated_rows_tie_to_the_smaller_index(metric):
    a, base = _operands(100, 300, 320, metric, seed=3)
    x = base.repeat_interleave(torch.randint(1, 9, (300,), generator=torch.Generator().manual_seed(1)).to(DEV), 0)
    x = x.contiguous()
    s, i, alpha, beta = _run(a, x, 50, metric)
    ref.check_chunked(s, i, a, x, alpha, beta)
    # within a block of equal rows the returned ones are the block's first
    first = torch.zeros(x.shape[0], dtype=torch.int64, device=DEV)
    same = (x[1:] == x[:-1]).all(1)
    for j in range(1, x.shape[0]):
        first[j] = first[j - 1] if bool(same[j - 1]) else j
    got = i.cpu()
    first = first.cpu()
    for q in range(got.shape[0]):
        chosen = set(got[q].tolist())
        for j in chosen:
            assert all(jj in chosen for jj in range(int(first[j]), j)), (q, j)


@pytest.mark.parametrize("offset", [0, 3, 997])
def test_self_offset_leaves_one_candidate_out(offset):
    """Query i is database row i + offset (while that exists), so the left-out candidate would be the best one."""
    a, x = _operands(1000, 1000, 320, "cosine", seed=offset)
    x[offset:] = a[: 1000 - offset]
    s, i, alpha, beta = _run(a, x, 10, "cosine", self_offset=offset)
    rows = torch.arange(1000, device=DEV)[:, None]
    assert not bool((i == rows + offset).any())
    ref.check_chunked(s, i, a, x, alpha, beta, self_offset=offset)


def test_search_all_leaves_each_row_out():
    from esm_b200 import search
    g = torch.Generator().manual_seed(2)
    for metric in ("cosine", "l2"):
        index = search.EmbeddingIndex(torch.randn(3000, 480, generator=g), metric=metric).to(DEV)
        s, i = index.search_all(k=10)
        assert not bool((i == torch.arange(3000, device=DEV)[:, None]).any())
        ks, ki, alpha, beta = _run(index.rows, index.rows, 10, metric, self_offset=0)
        assert torch.equal(ki, i)
        ref.check_chunked(ks, ki, index.rows, index.rows, alpha, beta, self_offset=0)


# ---- 3. invariance -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_outputs_do_not_depend_on_splits_batching_or_query_order(metric):
    a, x = _operands(300, 30_000, 512, metric, seed=9)
    tiles = -(-30_000 // 256)
    s, i, _, _ = _run(a, x, 64, metric, splits=1)
    for sp in (3, 7, min(1024, tiles)):
        s2, i2, _, _ = _run(a, x, 64, metric, splits=sp)
        assert torch.equal(s, s2) and torch.equal(i, i2), sp
    perm = torch.randperm(300, generator=torch.Generator().manual_seed(0)).to(DEV)
    s3, i3, _, _ = _run(a[perm].contiguous(), x, 64, metric)
    assert torch.equal(s3, s[perm]) and torch.equal(i3, i[perm])
    for b0, b1 in ((0, 1), (1, 64), (64, 65), (65, 300)):
        s4, i4, _, _ = _run(a[b0:b1].contiguous(), x, 64, metric)
        assert torch.equal(s4, s[b0:b1]) and torch.equal(i4, i[b0:b1])
    # the index's batched search equals one call
    from esm_b200 import search
    index = search.EmbeddingIndex._from_rows(x, 512, None, metric, None)
    old = search.QUERY_BATCH
    try:
        search.QUERY_BATCH = 64
        sb, ib = index._search_rows(a, 64, self_rows=False)
    finally:
        search.QUERY_BATCH = old
    sf, if_ = index._search_rows(a, 64, self_rows=False)
    assert torch.equal(sb, sf) and torch.equal(ib, if_) and torch.equal(if_, i)


# ---- 4. refusals -------------------------------------------------------------------------------------------------------
def test_every_refusal_launches_nothing():
    from esm_b200 import _lib
    lib = _lib.load()
    a, x = _operands(8, 300, 320, "cosine", seed=0)
    out_s = torch.empty(8, 128, device=DEV)
    out_i = torch.empty(8, 128, dtype=torch.int64, device=DEV)
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    P = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    base = dict(queries=P(a), q_ld=320, Q=8, base=P(x), b_ld=320, N=300, D=320, beta=None, alpha=1.0,
                self_offset=-1, k=10, splits=2, scratch=P(scratch), scratch_bytes=1 << 20, out_scores=P(out_s),
                out_idx=P(out_i))
    cases = [
        ({"queries": None}, "null"), ({"base": None}, "null"), ({"scratch": None}, "null"),
        ({"out_scores": None}, "null"), ({"out_idx": None}, "null"),
        ({"k": 0}, "1 <= k <= 128"), ({"k": 129}, "1 <= k <= 128"),
        ({"N": 5, "k": 6}, "candidates"), ({"self_offset": 0, "N": 10, "k": 10}, "candidates"),
        ({"D": 100}, "D % 64"), ({"D": 0}, "D % 64"),
        ({"q_ld": 300}, "q_ld"), ({"b_ld": 324}, "b_ld"),
        ({"queries": ctypes.c_void_p(a.data_ptr() + 8)}, "16-byte aligned"),
        ({"splits": 0}, "splits"), ({"splits": 1025}, "splits"),
        ({"scratch_bytes": 8 * 2 * 10 * 8 - 1}, "scratch smaller"),
        ({"Q": -1}, "Q >= 0"), ({"N": 0}, "N < 2^31"), ({"N": 1 << 31}, "N < 2^31"),
    ]
    torch.cuda.synchronize()
    for over, msg in cases:
        kw = dict(base, **over)
        before = lib.esmb200_launch_count()
        rc = lib.esmb200_knn_search(*kw.values(), None)
        assert rc == -1 and msg in lib.esmb200_last_error().decode(), (over, lib.esmb200_last_error())
        assert lib.esmb200_launch_count() == before
    before = lib.esmb200_launch_count()
    assert lib.esmb200_knn_search(*base.values(), None) == 0
    assert lib.esmb200_launch_count() == before + 2
    torch.cuda.synchronize()


def test_python_refusals_come_before_any_launch():
    from esm_b200 import _lib, search
    index = search.EmbeddingIndex(torch.randn(50, 320), metric="cosine").to(DEV)
    before = _lib.load().esmb200_launch_count()
    for bad, err in (((torch.randn(3, 64),), ValueError), ((torch.full((3, 320), float("nan")),), ValueError),
                     ((torch.zeros(3, 320),), ValueError)):
        with pytest.raises(err):
            index.search(*bad, k=5)
    for k in (0, 51, 129):
        with pytest.raises(ValueError):
            index.search(torch.randn(2, 320), k=k)
    with pytest.raises(ValueError):
        index.search_all(k=50)
    assert _lib.load().esmb200_launch_count() == before


# ---- 5. the command line ---------------------------------------------------------------------------------------------
def _write_extract_dir(root, labels, vecs, layer):
    for label, v in zip(labels, vecs):
        path = root / f"{label}.pt"
        path.parent.mkdir(parents=True, exist_ok=True)
        torch.save({"label": label, "mean_representations": {layer: v.clone()}}, path)


@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_cli_build_and_query_give_the_api_hits(tmp_path, metric):
    from esm_b200 import search, search_cli
    g = torch.Generator().manual_seed(4)
    db_labels = [f"fam{i % 7}/p{i:04d}" for i in range(700)]
    q_labels = [f"q{i:02d}" for i in range(20)]  # label order is file order
    xv, qv = torch.randn(700, 480, generator=g), torch.randn(20, 480, generator=g)
    _write_extract_dir(tmp_path / "db", db_labels, xv, 12)
    _write_extract_dir(tmp_path / "q", q_labels, qv, 12)
    p = search_cli.create_parser()
    assert search_cli.run(p.parse_args(["build", str(tmp_path / "db"), "--layer", "12", "--metric", metric,
                                        "--out", str(tmp_path / "db.pt")])) == 700
    n = search_cli.run(p.parse_args(["query", str(tmp_path / "db.pt"), "--queries", str(tmp_path / "q"), "--k", "5",
                                     "--out", str(tmp_path / "hits.tsv")]))
    assert n == 100
    order = sorted(range(700), key=lambda i: db_labels[i])
    index = search.EmbeddingIndex(xv[order].to(DEV), [db_labels[i] for i in order], metric)
    s, i = index.search(qv, k=5)
    lines = (tmp_path / "hits.tsv").read_text().splitlines()
    assert lines[0] == "query\trank\ttarget\tscore"
    want = [f"{q}\t{r + 1}\t{index.labels[j]}\t{v:.6g}" for q, rs, ri in zip(q_labels, s.tolist(), i.tolist())
            for r, (v, j) in enumerate(zip(rs, ri))]
    assert lines[1:] == want
    n = search_cli.run(p.parse_args(["query", str(tmp_path / "db.pt"), "--all", "--k", "3",
                                     "--out", str(tmp_path / "all.tsv")]))
    s, i = index.search_all(k=3)
    lines = (tmp_path / "all.tsv").read_text().splitlines()[1:]
    assert n == 2100 and lines == [f"{q}\t{r + 1}\t{index.labels[j]}\t{v:.6g}" for q, rs, ri in
                                   zip(index.labels, s.tolist(), i.tolist()) for r, (v, j) in enumerate(zip(rs, ri))]
