"""GPU: streamed search over sharded indexes (esm_b200.search.ShardedIndex, esmb200_knn_search_accumulate,
esmb200_knn_decode).

  1. ShardedIndex.search / search_all equal EmbeddingIndex.search / search_all bit for bit (torch.equal on scores and
     indices): both metrics, k in {1, 10, 128}, N not a multiple of 256, chunks of one tile, an odd number of tiles and
     the whole database, several shards, and more queries than QUERY_BATCH;
  2. duplicated rows in different chunks and shards tie to the smaller global index; the self row is left out when it
     sits at a chunk boundary;
  3. the accumulate / decode pair against the float64 restatement (tests/search_refs.py);
  4. device memory stays under max_device_bytes with a database five times larger, and a short last query batch
     that needs more scratch than a full one;
  5. every C-ABI refusal with real buffers, and every tensor check of the Python helpers, launching nothing;
  6. search_cli query on a directory index writes the hits.tsv of the .pt index built from the same extract directory.
Sizes stay at tens of thousands of rows.
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


def _vecs(n, E, seed):
    return torch.randn(n, E, generator=torch.Generator().manual_seed(seed))


def _write(path, x, metric, shard_rows, labels=None):
    from esm_b200 import search
    with search.IndexWriter(path, x.shape[1], metric, shard_rows=shard_rows) as w:
        w.add(x, labels)
    return search.ShardedIndex.open(path)


def _cap_for_chunk(index, q_rows, q_out, k, tiles):
    """max_device_bytes whose plan gives chunks of `tiles` 256-row tiles."""
    from esm_b200 import search
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cap = search.device_bytes(q_rows, q_out, k, index.padded_dim, index.metric, 256 * tiles, sms)
    assert search.plan_chunk_rows(q_rows, q_out, k, index.padded_dim, index.metric, cap, sms) == 256 * tiles
    return cap


# ---- 1. the resident index's results, bit for bit ------------------------------------------------------------------
N1, E1, Q1 = 5037, 320, 300


@pytest.fixture(scope="module")
def pair(tmp_path_factory):
    from esm_b200 import search
    root = tmp_path_factory.mktemp("shards")
    x = _vecs(N1, E1, 1)
    out = {}
    for metric in ("cosine", "l2"):
        out[metric] = (_write(root / metric, x, metric, shard_rows=1500),
                       search.EmbeddingIndex(x, metric=metric).to(DEV))
    return out


@pytest.mark.parametrize("metric", ["cosine", "l2"])
@pytest.mark.parametrize("k", [1, 10, 128])
@pytest.mark.parametrize("tiles", [1, 5, None])  # None: the default cap, one chunk for the whole database
def test_search_equals_the_resident_index(pair, metric, k, tiles, monkeypatch):
    from esm_b200 import search
    sharded, resident = pair[metric]
    assert len(sharded.shards) == 4
    queries = _vecs(Q1, E1, 2)
    s0, i0 = resident.search(queries, k)
    cap = None if tiles is None else _cap_for_chunk(sharded, Q1, Q1, k, tiles)
    s, i = sharded.search(queries, k, max_device_bytes=cap)
    assert s.device.type == "cuda" and i.dtype == torch.int64
    assert torch.equal(s, s0) and torch.equal(i, i0)
    monkeypatch.setattr(search, "QUERY_BATCH", 64)  # more queries than one batch (more stripes: a new cap)
    cap = None if tiles is None else _cap_for_chunk(sharded, Q1, Q1, k, tiles)
    s, i = sharded.search(queries, k, max_device_bytes=cap)
    assert torch.equal(s, s0) and torch.equal(i, i0)
    s, i = sharded.search(queries[7], k, max_device_bytes=None if tiles is None else
                          _cap_for_chunk(sharded, 1, 1, k, tiles))  # one query, [E]
    assert torch.equal(s, s0[7:8]) and torch.equal(i, i0[7:8])


@pytest.mark.parametrize("metric", ["cosine", "l2"])
@pytest.mark.parametrize("k", [1, 10, 128])
@pytest.mark.parametrize("tiles", [1, 5, None])
def test_search_all_equals_the_resident_index(pair, metric, k, tiles, monkeypatch):
    from esm_b200 import search
    sharded, resident = pair[metric]
    s0, i0 = resident.search_all(k)
    cap = None if tiles is None else _cap_for_chunk(sharded, N1, N1, k, tiles)
    s, i = sharded.search_all(k, max_device_bytes=cap)
    assert torch.equal(s, s0) and torch.equal(i, i0)
    if tiles == 5:
        monkeypatch.setattr(search, "QUERY_BATCH", 1024)
        s, i = sharded.search_all(k, max_device_bytes=_cap_for_chunk(sharded, N1, N1, k, tiles))
        assert torch.equal(s, s0) and torch.equal(i, i0)


def test_search_all_in_query_blocks_equals_the_resident_index(pair):
    """A cap too small for every query row at once: search_all takes the database's rows as queries block by block."""
    from esm_b200 import search
    sharded, resident = pair["l2"]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cap = 2 * search._fixed_device_bytes(1024, N1, 10, sharded.padded_dim, "l2", sms)
    assert sharded._query_block(10, cap, sms) < N1
    s0, i0 = resident.search_all(10)
    s, i = sharded.search_all(10, max_device_bytes=cap)
    assert torch.equal(s, s0) and torch.equal(i, i0)


@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_a_short_last_batch_that_needs_more_scratch(pair, metric, monkeypatch):
    """Q = 1,853 in batches of 1,024 on 132 SMs: the 829-query last batch runs 21 stripes (17,409 query-stripes)
    against the first batch's 17 (17,408), so scratch sized for the first batch would be too small."""
    from esm_b200 import search
    sharded, resident = pair[metric]
    monkeypatch.setattr(search, "QUERY_BATCH", 1024)
    queries = _vecs(1853, E1, 16)
    s0, i0 = resident.search(queries, 10)
    s, i = sharded.search(queries, 10)
    assert torch.equal(s, s0) and torch.equal(i, i0)


# ---- 2. ties and the self row --------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_duplicated_rows_across_chunks_and_shards_tie_to_the_smaller_index(tmp_path, metric):
    from esm_b200 import search
    base = _vecs(300, 320, 3)
    x = torch.cat([base, base.flip(0), base, base[:97]])  # each row 3-4 times, in different chunks and shards
    sharded = _write(tmp_path / "db", x, metric, shard_rows=333)
    resident = search.EmbeddingIndex(x, metric=metric).to(DEV)
    q = torch.cat([base[:50], _vecs(50, 320, 4)])
    cap = _cap_for_chunk(sharded, 100, 100, 40, 1)
    s, i = sharded.search(q, 40, max_device_bytes=cap)
    s0, i0 = resident.search(q, 40)
    assert torch.equal(s, s0) and torch.equal(i, i0)
    rows = resident.rows.cpu()
    for qi in range(i.shape[0]):
        chosen = set(i[qi].tolist())
        for j in chosen:  # a copy is returned only after every smaller copy of the same row
            copies = [jj for jj in range(j) if torch.equal(rows[jj], rows[j])]
            assert all(jj in chosen for jj in copies), (qi, j)
    assert bool((i[:50, 0] == torch.arange(50, device=DEV)).all())  # the exact row, at its first copy


@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_the_self_row_is_left_out_at_chunk_boundaries(tmp_path, metric):
    from esm_b200 import search
    x = _vecs(1100, 320, 5)
    for a, b in ((255, 256), (511, 512), (767, 768)):  # twins on either side of a one-tile chunk boundary
        x[b] = x[a]
    sharded = _write(tmp_path / "db", x, metric, shard_rows=400)
    resident = search.EmbeddingIndex(x, metric=metric).to(DEV)
    cap = _cap_for_chunk(sharded, 1100, 1100, 10, 1)
    s, i = sharded.search_all(10, max_device_bytes=cap)
    s0, i0 = resident.search_all(10)
    assert torch.equal(s, s0) and torch.equal(i, i0)
    assert not bool((i == torch.arange(1100, device=DEV)[:, None]).any())
    for a, b in ((255, 256), (511, 512), (767, 768)):
        assert int(i[a, 0]) == b and int(i[b, 0]) == a


# ---- 3. the kernel pair against the float64 restatement -----------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "l2"])
@pytest.mark.parametrize("k,chunk", [(1, 256), (37, 768), (128, 1280)])
def test_accumulate_and_decode_match_the_float64_restatement(metric, k, chunk):
    from esm_b200 import search
    g = torch.Generator().manual_seed(k + chunk)
    a = search.prepare_rows(torch.randn(200, 1280, generator=g), metric).to(DEV)
    x = search.prepare_rows(torch.randn(10_001, 1280, generator=g), metric).to(DEV)
    beta = -search.squared_norms(x) if metric == "l2" else None
    alpha = 2.0 if metric == "l2" else 1.0
    for self_offset in (-1, 0):
        keys = torch.zeros((200, k), dtype=torch.int64, device=DEV)
        for g0 in range(0, 10_001, chunk):
            g1 = min(10_001, g0 + chunk)
            search.knn_accumulate(a if self_offset < 0 else x[:200], x[g0:g1], g0, k, keys, None,
                                  None if beta is None else beta[g0:g1].contiguous(), alpha, self_offset)
        s = torch.empty((200, k), device=DEV)
        i = torch.empty((200, k), dtype=torch.int64, device=DEV)
        search.knn_decode(keys, s, i)
        q = a if self_offset < 0 else x[:200]
        ref.check_chunked(s, i, q, x, alpha, beta, self_offset=self_offset)
        s0, i0 = search.knn(q, x, k, beta, alpha, self_offset)
        assert torch.equal(s, s0) and torch.equal(i, i0)


# ---- 4. device memory --------------------------------------------------------------------------------------------
def test_device_memory_stays_under_the_cap(tmp_path):
    from esm_b200 import search
    x = _vecs(40_000, 1280, 6)
    sharded = _write(tmp_path / "db", x, "l2", shard_rows=15_000)
    db_bytes = 40_000 * 1280 * 2
    cap = db_bytes // 5
    q = _vecs(100, 1280, 7)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    s, i = sharded.search(q, 10, max_device_bytes=cap)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - before <= cap
    del s, i
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    s, i = sharded.search_all(10, max_device_bytes=cap)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - before <= cap
    resident = search.EmbeddingIndex(x, metric="l2").to(DEV)
    s0, i0 = resident.search_all(10)
    assert torch.equal(s, s0) and torch.equal(i, i0)


# ---- 5. refusals ---------------------------------------------------------------------------------------------------
def test_every_refusal_launches_nothing():
    from esm_b200 import _lib, search
    lib = _lib.load()
    a = search.prepare_rows(_vecs(8, 320, 8), "cosine").to(DEV)
    x = search.prepare_rows(_vecs(300, 320, 9), "cosine").to(DEV)
    keys = torch.zeros(8, 128, dtype=torch.int64, device=DEV)
    out_s = torch.empty(8, 128, device=DEV)
    out_i = torch.empty(8, 128, dtype=torch.int64, device=DEV)
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    P = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)  # noqa: E731
    acc = dict(queries=P(a), q_ld=320, Q=8, base=P(x), b_ld=320, n=300, row0=1000, D=320, beta=None, alpha=1.0,
               self_offset=-1, k=10, splits=2, scratch=P(scratch), scratch_bytes=1 << 20, keys=P(keys))
    cases = [
        ({"queries": None}, "null"), ({"base": None}, "null"), ({"scratch": None}, "null"), ({"keys": None}, "null"),
        ({"k": 0}, "1 <= k <= 128"), ({"k": 129}, "1 <= k <= 128"),
        ({"D": 100}, "D % 64"), ({"D": 0}, "D % 64"), ({"q_ld": 300}, "q_ld"), ({"b_ld": 324}, "b_ld"),
        ({"queries": P(a, 8)}, "16-byte aligned"), ({"keys": P(keys, 4)}, "8-byte aligned"),
        ({"splits": 0}, "splits"), ({"splits": 1025}, "splits"),
        ({"scratch_bytes": 8 * 2 * 10 * 8 - 1}, "scratch smaller"),
        ({"Q": -1}, "Q >= 0"), ({"n": 0}, "n >= 1"), ({"row0": -1}, "row0 >= 0"),
        ({"row0": (1 << 31) - 300}, "row0 + n < 2^31"),
    ]
    torch.cuda.synchronize()
    for over, msg in cases:
        kw = dict(acc, **over)
        before = lib.esmb200_launch_count()
        rc = lib.esmb200_knn_search_accumulate(*kw.values(), None)
        assert rc == -1 and msg in lib.esmb200_last_error().decode(), (over, lib.esmb200_last_error())
        assert lib.esmb200_launch_count() == before
    dec = dict(keys=P(keys), Q=8, k=10, out_scores=P(out_s), out_idx=P(out_i))
    for over, msg in [({"keys": None}, "null"), ({"out_scores": None}, "null"), ({"out_idx": None}, "null"),
                      ({"keys": P(keys, 4)}, "8-byte aligned"), ({"out_scores": P(out_s, 2)}, "4-byte aligned"),
                      ({"out_idx": P(out_i, 4)}, "8-byte aligned out_idx"), ({"Q": -1}, "Q >= 0"),
                      ({"k": 0}, "1 <= k"), ({"k": 129}, "1 <= k")]:
        kw = dict(dec, **over)
        before = lib.esmb200_launch_count()
        assert lib.esmb200_knn_decode(*kw.values(), None) == -1 and msg in lib.esmb200_last_error().decode()
        assert lib.esmb200_launch_count() == before
    before = lib.esmb200_launch_count()
    assert lib.esmb200_knn_search_accumulate(*acc.values(), None) == 0
    assert lib.esmb200_launch_count() == before + 2
    assert lib.esmb200_knn_decode(*dec.values(), None) == 0
    assert lib.esmb200_launch_count() == before + 3
    assert lib.esmb200_knn_search_accumulate(*dict(acc, Q=0).values(), None) == 0
    assert lib.esmb200_knn_decode(*dict(dec, Q=0).values(), None) == 0
    assert lib.esmb200_launch_count() == before + 3
    torch.cuda.synchronize()
    # every row of the chunk carries its global index
    s = torch.empty(8, 10, device=DEV)
    i = torch.empty(8, 10, dtype=torch.int64, device=DEV)
    search.knn_decode(keys.view(-1)[:80].view(8, 10), s, i)
    assert int(i.min()) >= 1000 and int(i.max()) < 1300


def test_the_host_ring_is_kept_between_calls_and_released(pair):
    from esm_b200 import search
    sharded, resident = pair["l2"]
    q = _vecs(20, E1, 19)
    s0, i0 = resident.search(q, 10)
    search.release_host_memory()
    s1, i1 = sharded.search(q, 10)
    rings = list(search._host_rings.values())
    assert len(rings) == 1 and rings[0]._registered
    s2, i2 = sharded.search(q, 10)
    assert list(search._host_rings.values())[0] is rings[0]  # reused, not registered again
    search.release_host_memory()
    assert not search._host_rings and not rings[0]._registered
    for s, i in ((s1, i1), (s2, i2)):
        assert torch.equal(s, s0) and torch.equal(i, i0)


def test_the_kernel_helpers_check_their_tensors():
    from esm_b200 import _lib, search
    a = search.prepare_rows(_vecs(8, 320, 17), "l2").to(DEV)
    x = search.prepare_rows(_vecs(300, 320, 18), "l2").to(DEV)
    beta = -search.squared_norms(x)
    keys = torch.zeros(8, 10, dtype=torch.int64, device=DEV)
    s = torch.empty(8, 10, device=DEV)
    i = torch.empty(8, 10, dtype=torch.int64, device=DEV)
    lib = _lib.load()
    torch.cuda.synchronize()
    before = lib.esmb200_launch_count()
    bad_acc = [dict(keys=keys.int()), dict(keys=torch.zeros(10, 8, dtype=torch.int64, device=DEV).T),
               dict(keys=keys[:, :5]), dict(keys=keys.cpu()), dict(beta=beta[:299]), dict(beta=beta.double()),
               dict(queries=a.float()), dict(base=x.cpu()), dict(queries=a[:, :256].contiguous()),
               dict(scratch=torch.empty(1 << 16, dtype=torch.int32, device=DEV))]
    for over in bad_acc:
        kw = dict(queries=a, base=x, row0=0, k=10, keys=keys, scratch=None, beta=beta, alpha=2.0)
        kw.update(over)
        with pytest.raises(ValueError):
            search.knn_accumulate(**kw)
    for over in (dict(keys=keys.int()), dict(keys=keys.T), dict(scores=s.double()), dict(scores=s[:4]),
                 dict(idx=i.int()), dict(idx=torch.empty(10, 8, dtype=torch.int64, device=DEV).T)):
        kw = dict(keys=keys, scores=s, idx=i)
        kw.update(over)
        with pytest.raises(ValueError):
            search.knn_decode(**kw)
    assert lib.esmb200_launch_count() == before
    search.knn_accumulate(a, x, 0, 10, keys, None, beta, 2.0)
    search.knn_decode(keys, s, i)
    s0, i0 = search.knn(a, x, 10, beta, 2.0)
    assert torch.equal(s, s0) and torch.equal(i, i0)


def test_python_refusals_come_before_any_launch(tmp_path):
    from esm_b200 import _lib
    sharded = _write(tmp_path / "db", _vecs(50, 320, 10), "cosine", shard_rows=20)
    before = _lib.load().esmb200_launch_count()
    for bad in (torch.randn(3, 64), torch.full((3, 320), float("nan")), torch.zeros(3, 320)):
        with pytest.raises(ValueError):
            sharded.search(bad, k=5)
    for k in (0, 51, 129):
        with pytest.raises(ValueError):
            sharded.search(torch.randn(2, 320), k=k)
    with pytest.raises(ValueError):
        sharded.search_all(k=50)
    with pytest.raises(ValueError, match="leaves no room"):
        sharded.search(torch.randn(2, 320), k=5, max_device_bytes=1000)
    with pytest.raises(ValueError, match="CUDA device"):
        sharded.search(torch.randn(2, 320), k=5, device="cpu")
    assert _lib.load().esmb200_launch_count() == before


# ---- 6. the command line -------------------------------------------------------------------------------------------
def _write_extract_dir(root, labels, vecs, layer):
    for label, v in zip(labels, vecs):
        path = root / f"{label}.pt"
        path.parent.mkdir(parents=True, exist_ok=True)
        torch.save({"label": label, "mean_representations": {layer: v.clone()}}, path)


@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_cli_query_on_a_directory_writes_the_pt_hits(tmp_path, metric):
    from esm_b200 import search_cli
    g = torch.Generator().manual_seed(4)
    db_labels = [f"fam{i % 7}/p{(i * 31) % 700:04d}" for i in range(700)]
    q_labels = [f"q{i:02d}" for i in range(20)]
    _write_extract_dir(tmp_path / "db", db_labels, torch.randn(700, 480, generator=g), 12)
    _write_extract_dir(tmp_path / "q", q_labels, torch.randn(20, 480, generator=g), 12)
    p = search_cli.create_parser()
    for out in ("db.pt", "dbdir"):
        assert search_cli.run(p.parse_args(["build", str(tmp_path / "db"), "--layer", "12", "--metric", metric,
                                            "--out", str(tmp_path / out), "--shard-rows", "300"])) == 700
    for out in ("db.pt", "dbdir"):
        n = search_cli.run(p.parse_args(["query", str(tmp_path / out), "--queries", str(tmp_path / "q"), "--k", "5",
                                         "--out", str(tmp_path / f"{out}.hits.tsv")]))
        assert n == 100
        n = search_cli.run(p.parse_args(["query", str(tmp_path / out), "--all", "--k", "3",
                                         "--out", str(tmp_path / f"{out}.all.tsv")]))
        assert n == 2100
    for kind in ("hits", "all"):
        a = (tmp_path / f"db.pt.{kind}.tsv").read_text()
        b = (tmp_path / f"dbdir.{kind}.tsv").read_text()
        assert a == b and len(a.splitlines()) > 100
