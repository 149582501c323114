"""CPU: the inverted-file index (esm_b200.search.IVFIndex) without a GPU. The new C symbols, the scratch sizes as host
arithmetic, the C-ABI refusals with placeholder pointers, the exact k-means mean reference, the empty-cluster rule,
the training sample, the save / load round trip and the CLI's IVF options and refusals."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import ivf_refs  # noqa: E402

ROOT = os.path.dirname(HERE)
SYMBOLS = ("esmb200_ivf_scratch_bytes", "esmb200_ivf_search", "esmb200_kmeans_means")


def test_new_symbols_are_declared_and_exported_at_abi_4():
    from esm_b200 import _lib
    header = open(os.path.join(ROOT, "include", "esmb200.h")).read()
    lib = _lib.load()
    assert lib.esmb200_abi_version() == 4
    for name in SYMBOLS:
        assert f"int {name}(" in header, name
        assert name in _lib.EXPORTS, name
        assert hasattr(lib, name), name


def _scratch(Q, nprobe, nlist, N, D, k):
    from esm_b200 import search
    return search.ivf_scratch_bytes(Q, nprobe, nlist, N, D, k)


def test_scratch_sizes_are_host_arithmetic():
    # no device is touched: the sizes follow from the arguments alone
    Q, nprobe, nlist, N, D, k = 1000, 32, 4096, 10_000_000, 1280, 10
    b = _scratch(Q, nprobe, nlist, N, D, k)
    assert b % 256 == 0
    assert b >= Q * nprobe * D * 2 + Q * (nprobe + 64) * k * 8  # gathered rows and the partial lists
    assert b < Q * nprobe * D * 2 + Q * (nprobe + 64) * k * 8 + 40 * Q * nprobe + 64 * nlist + 24 * (Q + 64 * 64) + 4096
    assert _scratch(2 * Q, nprobe, nlist, N, D, k) > b
    # every list: no gathered rows, a few stripes per query
    assert _scratch(Q, nlist, nlist, N, D, k) < Q * 20 * k * 8 + 4096 * 20
    assert _scratch(0, 8, 16, 100, 64, 1) >= 256
    from esm_b200 import search
    assert 1 <= search.ivf_query_batch(128, 4096, N, D, 128) < search.QUERY_BATCH
    assert search.ivf_query_batch(8, 4096, 100_000, 64, 1) == search.QUERY_BATCH
    n = search.ivf_query_batch(128, 4096, N, D, 128)
    assert _scratch(n, 128, 4096, N, D, 128) <= search.IVF_SCRATCH_CAP < _scratch(n + 1, 128, 4096, N, D, 128)


@pytest.mark.parametrize("over,msg", [
    ({"k": 0}, "1 <= k <= 128"), ({"k": 129}, "1 <= k <= 128"), ({"Q": -1}, "Q >= 0"), ({"N": 0}, "N < 2^31"),
    ({"N": 1 << 31}, "N < 2^31"), ({"nlist": 0}, "nlist"), ({"nlist": 200, "N": 100}, "nlist"),
    ({"nprobe": 0}, "nprobe"), ({"nprobe": 129, "nlist": 200, "N": 1000}, "nprobe"), ({"nprobe": 17}, "nprobe"),
    ({"D": 100}, "D % 64"), ({"Q": 1 << 24, "nprobe": 128, "nlist": 200, "N": 1000}, "Q * nprobe"),
    # int32 partial-list indices: 34 M queries of one probe have 34 M * 65 > 2^31 lists
    ({"Q": 34_000_000, "nprobe": 1, "nlist": 16, "N": 1000}, "Q * R < 2^31"),
])
def test_scratch_bytes_refusals(over, msg):
    from esm_b200 import _lib
    kw = dict(Q=8, nprobe=4, nlist=16, N=300, D=64, k=10)
    kw.update(over)
    out = ctypes.c_size_t(0)
    rc = _lib.load().esmb200_ivf_scratch_bytes(*kw.values(), ctypes.byref(out))
    assert rc == -1 and msg in _lib.load().esmb200_last_error().decode()


# Placeholder pointers, which a refused call never dereferences; these run only where no CUDA device is present, and
# tests/test_gpu_ivf.py repeats every refusal with real buffers.
_FAKE = 4096
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="placeholder pointers: only where nothing can launch")
IVF_ARGS = dict(queries=_FAKE, q_ld=64, Q=8, rows=_FAKE, b_ld=64, N=300, ids=_FAKE, offsets=_FAKE, nlist=16, D=64,
                beta=None, alpha=1.0, probes=_FAKE, nprobe=4, self_ids=None, k=10, scratch=_FAKE,
                scratch_bytes=1 << 24, out_scores=_FAKE, out_idx=_FAKE)
IVF_REFUSALS = [
    ({"queries": None}, "null"), ({"rows": None}, "null"), ({"ids": None}, "null"), ({"offsets": None}, "null"),
    ({"scratch": None}, "null"), ({"out_scores": None}, "null"), ({"out_idx": None}, "null"),
    ({"probes": None}, "probes NULL exactly"), ({"nprobe": 16}, "probes NULL exactly"),
    ({"k": 0}, "1 <= k <= 128"), ({"k": 129}, "1 <= k <= 128"), ({"Q": -1}, "Q >= 0"), ({"N": 0}, "N < 2^31"),
    ({"nlist": 0}, "nlist"), ({"nprobe": 0}, "nprobe"), ({"nprobe": 17}, "nprobe"), ({"D": 96}, "D % 64"),
    ({"q_ld": 60}, "q_ld"), ({"b_ld": 68}, "b_ld"), ({"queries": _FAKE + 8}, "16-byte aligned"),
    ({"rows": _FAKE + 2}, "16-byte aligned"), ({"ids": _FAKE + 4}, "8-byte aligned"),
    ({"self_ids": _FAKE + 4}, "8-byte aligned"), ({"probes": _FAKE + 2}, "4-byte aligned probes"),
    ({"out_idx": _FAKE + 4}, "8-byte aligned out_idx"), ({"scratch": _FAKE + 16}, "256-byte aligned"),
    ({"scratch_bytes": 256}, "scratch smaller"), ({"Q": 34_000_000, "nprobe": 1}, "Q * R < 2^31"),
]


@no_device
@pytest.mark.parametrize("over,msg", IVF_REFUSALS, ids=lambda v: v if isinstance(v, str) else "-".join(v) if isinstance(v, dict) else "")
def test_ivf_search_refuses_bad_arguments(over, msg):
    from esm_b200 import _lib
    lib = _lib.load()
    kw = dict(IVF_ARGS, **over)
    before = lib.esmb200_launch_count()
    rc = lib.esmb200_ivf_search(*kw.values(), None)
    assert rc == -1 and msg in lib.esmb200_last_error().decode(), lib.esmb200_last_error()
    assert lib.esmb200_launch_count() == before


MEANS_ARGS = dict(rows=_FAKE, ld=64, n=100, D=64, assign=_FAKE, nlist=4, sums=_FAKE, means=_FAKE, counts=_FAKE)
MEANS_REFUSALS = [
    ({"rows": None}, "null"), ({"assign": None}, "null"), ({"sums": None}, "null"), ({"means": None}, "null"),
    ({"counts": None}, "null"), ({"n": -1}, "n <= 2^23"), ({"n": (1 << 23) + 1}, "n <= 2^23"), ({"D": 12}, "D % 8"),
    ({"ld": 60}, "ld >= D"), ({"nlist": 0}, "nlist"), ({"rows": _FAKE + 8}, "16-byte aligned"),
    ({"assign": _FAKE + 4}, "8-byte aligned"),
]


@no_device
@pytest.mark.parametrize("over,msg", MEANS_REFUSALS, ids=lambda v: v if isinstance(v, str) else "-".join(v) if isinstance(v, dict) else "")
def test_kmeans_means_refuses_bad_arguments(over, msg):
    from esm_b200 import _lib
    lib = _lib.load()
    kw = dict(MEANS_ARGS, **over)
    before = lib.esmb200_launch_count()
    rc = lib.esmb200_kmeans_means(*kw.values(), None)
    assert rc == -1 and msg in lib.esmb200_last_error().decode(), lib.esmb200_last_error()
    assert lib.esmb200_launch_count() == before


# ---- k-means pieces ---------------------------------------------------------------------------------------------------
def test_exact_mean_reference_on_a_hand_made_case():
    x = torch.tensor([[1.0, -2.0, 65504.0], [0.5, 2.0, 65504.0], [2 ** -24, 0.0, -1.0], [3.0, 3.0, 3.0]],
                     dtype=torch.float16)
    a = torch.tensor([0, 0, 0, 2])
    sums, means, counts = ivf_refs.exact_means(x, a, 4)
    assert counts.tolist() == [3, 0, 1, 0]
    assert sums[0].tolist() == [int((1.5 + 2 ** -24) * 2 ** 24), 0, (2 * 65504 - 1) * 2 ** 24]
    assert means[0, 0].item() == torch.tensor((1.5 + 2 ** -24) / 3, dtype=torch.float64).float().item()
    assert means[0, 2].item() == torch.tensor((2 * 65504 - 1) / 3, dtype=torch.float64).float().item()
    assert means[2].tolist() == [3.0, 3.0, 3.0] and means[1].tolist() == [0.0, 0.0, 0.0]
    # the order of the members does not matter: the sums are exact integers
    p = torch.tensor([2, 0, 3, 1])
    assert torch.equal(ivf_refs.exact_means(x[p], a[p], 4)[1], means)


def test_the_empty_cluster_rule_on_a_hand_made_case():
    from esm_b200 import search
    x = torch.arange(12, dtype=torch.float16).reshape(6, 2)
    cent = torch.full((4, 2), -1.0, dtype=torch.float16)
    s = torch.tensor([0.9, 0.2, 0.5, 0.2, 0.1, 0.7])   # cosine: lowest similarity first, ties to the smaller row
    assert search.worst_served(s, None, "cosine").tolist() == [4, 1, 3, 2, 5, 0]
    empty = torch.tensor([False, True, False, True])
    out = search.fill_empty(cent, empty, x, s, None, "cosine")
    assert torch.equal(out[1], x[4]) and torch.equal(out[3], x[1])
    assert torch.equal(out[0], cent[0]) and torch.equal(out[2], cent[2])
    # l2: the largest distance |x|^2 - s first
    xn = torch.tensor([5.0, 5.0, 1.0, 9.0, 2.0, 5.0])
    s2 = torch.tensor([1.0, 4.0, -3.0, 5.0, 1.0, 1.0])   # distances 4, 1, 4, 4, 1, 4
    assert search.worst_served(s2, xn, "l2").tolist() == [0, 2, 3, 5, 1, 4]
    out = search.fill_empty(cent, torch.tensor([True, False, False, False]), x, s2, xn, "l2")
    assert torch.equal(out[0], x[0])
    assert search.fill_empty(cent, torch.zeros(4, dtype=torch.bool), x, s, None, "cosine") is cent


def test_the_sum_bound_refuses_a_cluster_that_could_overflow():
    from esm_b200 import search
    search.check_sum_bound(torch.tensor([1 << 23, 5]), 65504.0)          # (2^16 - 32) 2^47 < 2^63
    search.check_sum_bound(torch.tensor([1 << 38]), 1.0)                 # cosine rows: 2^62
    with pytest.raises(ValueError, match="overflow"):
        search.check_sum_bound(torch.tensor([3, (1 << 23) + (1 << 13)]), 65504.0)  # just past 2^63 / (65504 2^24)
    with pytest.raises(ValueError, match="overflow"):
        search.check_sum_bound(torch.tensor([1 << 39]), 1.0)
    search.check_sum_bound(torch.zeros(0, dtype=torch.int64), 65504.0)


def test_the_training_sample_and_initial_centroids_follow_the_seed():
    from esm_b200 import search
    s = search.training_sample(1000, 300, 7)
    assert torch.equal(s, torch.randperm(1000, generator=torch.Generator().manual_seed(7))[:300])
    assert torch.equal(s, search.training_sample(1000, 300, 7))
    assert not torch.equal(s, search.training_sample(1000, 300, 8))
    assert len(set(s.tolist())) == 300


def _parts(N=50, E=70, nlist=4, metric="cosine", seed=0):
    from esm_b200 import search
    g = torch.Generator().manual_seed(seed)
    rows = search.prepare_rows(torch.randn(N, E, generator=g), metric)
    a = torch.randint(0, nlist, (N,), generator=g)
    ids = torch.sort(a, stable=True).indices
    offsets = torch.zeros(nlist + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.bincount(a, minlength=nlist), 0)
    cent = search.prepare_rows(torch.randn(nlist, E, generator=g), metric)
    return search.IVFIndex._from_parts(rows[ids], ids, offsets, cent, E, [f"p{i}" for i in range(N)], metric, 33,
                                       {"nlist": nlist, "train_rows": N, "iters": 3, "seed": 0})


@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_save_load_round_trip_on_the_cpu(tmp_path, metric):
    from esm_b200 import search
    index = _parts(metric=metric)
    index.save(tmp_path / "ivf.pt")
    back = search.IVFIndex.load(tmp_path / "ivf.pt", device="cpu")
    for name in ("rows", "ids", "offsets", "centroids"):
        assert torch.equal(getattr(back, name), getattr(index, name)), name
    assert (back.labels, back.metric, back.layer, back.dim, back.params, len(back)) == \
        (index.labels, metric, 33, 70, index.params, 50)
    assert back.device == torch.device("cpu")
    assert torch.equal(back._pos[back.ids], torch.arange(50))
    assert isinstance(search.load_file_index(tmp_path / "ivf.pt", device="cpu"), search.IVFIndex)
    with pytest.raises(ValueError, match="not a saved EmbeddingIndex"):
        search.EmbeddingIndex.load(tmp_path / "ivf.pt", device="cpu")
    search.EmbeddingIndex(torch.randn(5, 70)).save(tmp_path / "exact.pt")
    with pytest.raises(ValueError, match="not a saved IVFIndex"):
        search.IVFIndex.load(tmp_path / "exact.pt", device="cpu")
    assert isinstance(search.load_file_index(tmp_path / "exact.pt", device="cpu"), search.EmbeddingIndex)


def test_python_refusals_on_a_cpu_index():
    from esm_b200 import search
    index = _parts()
    for bad in (0, 5, 129, True, 2.0):
        with pytest.raises(ValueError, match="nprobe"):
            index.search(torch.randn(2, 70), k=3, nprobe=bad)
    assert index.check_nprobe(None) == 4 and index.check_nprobe(4) == 4
    with pytest.raises(ValueError, match="on the CPU"):
        index.search(torch.randn(2, 70), k=3, nprobe=2)
    with pytest.raises(ValueError, match="k must be"):
        index.search_all(k=50)
    x = torch.randn(20, 64)
    for kw, msg in (({"nlist": 0}, "nlist"), ({"nlist": 21}, "nlist"), ({"nlist": 4, "train_rows": 3}, "train_rows"),
                    ({"nlist": 4, "iters": -1}, "iters"), ({"nlist": 4, "seed": -1}, "seed")):
        with pytest.raises(ValueError, match=msg):
            search.IVFIndex(x, **kw)
    with pytest.raises(ValueError, match="labels"):
        search.IVFIndex(x, ["a"], nlist=2)


# ---- CLI ----------------------------------------------------------------------------------------------------------------
def test_cli_parses_the_ivf_options():
    from esm_b200 import search_cli
    p = search_cli.create_parser()
    a = p.parse_args(["build", "x/", "--layer", "33", "--out", "ivf.pt", "--nlist", "64", "--train-rows", "1000",
                      "--iters", "5", "--seed", "3"])
    assert (a.nlist, a.train_rows, a.iters, a.seed) == (64, 1000, 5, 3)
    a = p.parse_args(["build", "x/", "--layer", "33", "--out", "db.pt"])
    assert (a.nlist, a.train_rows, a.iters, a.seed) == (None, None, 20, 0)
    a = p.parse_args(["query", "ivf.pt", "--all", "--nprobe", "16", "--out", "h.tsv"])
    assert a.nprobe == 16
    assert p.parse_args(["query", "db.pt", "--all", "--out", "h.tsv"]).nprobe is None


@pytest.mark.parametrize("argv,msg", [
    (["--out", "{t}/db", "--nlist", "4"], "not a directory"),
    (["--out", "{t}/db.pt", "--nlist", "4", "--append"], "cannot --append"),
    (["--out", "{t}/db.pt", "--iters", "3"], "pass --nlist"),
])
def test_cli_build_refuses_nlist_with_a_directory_or_append(tmp_path, argv, msg):
    from esm_b200 import search_cli
    args = search_cli.create_parser().parse_args(
        ["build", str(tmp_path / "nothing"), "--layer", "33"] + [v.format(t=tmp_path) for v in argv])
    with pytest.raises(ValueError, match=msg):
        search_cli.run(args)
    assert not (tmp_path / "db").exists() and not (tmp_path / "db.pt").exists()


def test_cli_query_refuses_nprobe_on_an_exact_or_sharded_index(tmp_path):
    from esm_b200 import search, search_cli
    x = torch.randn(10, 64, generator=torch.Generator().manual_seed(1))
    search.EmbeddingIndex(x, layer=33).save(tmp_path / "db.pt")
    with search.IndexWriter(tmp_path / "db", dim=64, layer=33) as w:
        w.add(x)
    for index in ("db.pt", "db"):
        args = search_cli.create_parser().parse_args(
            ["query", str(tmp_path / index), "--all", "--nprobe", "2", "--out", str(tmp_path / "h.tsv")])
        with pytest.raises(ValueError, match="--nprobe applies to an IVF index"):
            search_cli.run(args)
    assert not (tmp_path / "h.tsv").exists()
    _parts(N=10, E=64).save(tmp_path / "ivf.pt")
    args = search_cli.create_parser().parse_args(
        ["query", str(tmp_path / "ivf.pt"), "--all", "--nprobe", "5", "--out", str(tmp_path / "h.tsv")])
    with pytest.raises(ValueError, match="nprobe must be"):
        search_cli.run(args)


def test_write_hits_skips_missing_slots(tmp_path):
    from esm_b200 import search_cli
    scores = torch.tensor([[0.9, float("nan")], [0.5, 0.4]])
    idx = torch.tensor([[1, -1], [0, 2]])
    n = search_cli.write_hits(tmp_path / "h.tsv", ["q0", "q1"], ["a", "b", "c"], scores, idx)
    assert n == 3
    assert (tmp_path / "h.tsv").read_text().splitlines() == [
        "query\trank\ttarget\tscore", "q0\t1\tb\t0.9", "q1\t1\ta\t0.5", "q1\t2\tc\t0.4"]
