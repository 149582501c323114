"""CPU: sharded search indexes (esm_b200.search.IndexWriter / ShardedIndex) without a GPU. The writer's round trip
(rows, labels and l2 norms bit for bit against prepare_rows / squared_norms, across shard boundaries), appending,
refusals of a mismatched index, a writer stopped before close(), the chunk planner's arithmetic, the CLI's new forms,
the Python refusals, the new symbols and the C-ABI refusals of esmb200_knn_search_accumulate / esmb200_knn_decode
with placeholder pointers."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def _vecs(n, E, seed):
    return torch.randn(n, E, generator=torch.Generator().manual_seed(seed))


def _read_all(index):
    out = np.empty((len(index), index.padded_dim), dtype=np.float16)
    beta = np.empty(len(index), dtype=np.float32) if index.metric == "l2" else None
    index.read_rows(0, len(index), out, beta)
    return torch.from_numpy(out), (None if beta is None else torch.from_numpy(beta))


# ---- the writer --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_writer_round_trip_is_bit_exact(tmp_path, metric):
    from esm_b200 import search
    x = _vecs(1000, 480, 1) * 3
    labels = [f"p|{i}/x" for i in range(1000)]
    with search.IndexWriter(tmp_path / "db", 480, metric, layer=12, shard_rows=300) as w:
        w.add(x[:10], labels[:10])
        w.add(x[10:777], labels[10:777])  # crosses two shard boundaries in one call
        w.add(x[777:], labels[777:])
    man = json.loads((tmp_path / "db" / "manifest.json").read_text())
    assert man["format"] == "esm_b200.search-shards/1" and man["padded_dim"] == 512 and man["layer"] == 12
    assert [s["rows"] for s in man["shards"]] == [300, 300, 300, 100]
    index = search.ShardedIndex.open(tmp_path / "db")
    ref = search.EmbeddingIndex(x, labels, metric, layer=12)
    assert len(index) == 1000 and index.dim == 480 and index.metric == metric and index.layer == 12
    rows, beta = _read_all(index)
    assert torch.equal(rows, ref.rows)
    assert list(index.labels) == labels and index.labels[999] == labels[999] and index.labels[300:302] == labels[300:302]
    if metric == "l2":
        assert torch.equal(-beta, ref.sqnorm)
        assert torch.equal(-beta, search.squared_norms(ref.rows))
    # one shard's bytes are the raw little-endian rows
    raw = np.fromfile(tmp_path / "db" / "shard-00001.f16", dtype="<f2").reshape(300, 512)
    assert torch.equal(torch.from_numpy(raw.astype(np.float16)), ref.rows[300:600])
    # a range read across shard boundaries at an offset
    part = np.empty((450, 512), dtype=np.float16)
    index.read_rows(250, 700, part)
    assert torch.equal(torch.from_numpy(part), ref.rows[250:700])


def test_append_adds_shards_after_the_existing_ones(tmp_path):
    from esm_b200 import search
    x = _vecs(500, 320, 2)
    with search.IndexWriter(tmp_path / "db", 320, "l2", layer=6, shard_rows=256) as w:
        w.add(x[:300])
    with search.IndexWriter(tmp_path / "db", 320, "l2", layer=6, shard_rows=256) as w:
        assert len(w) == 300
        w.add(x[300:])
    index = search.ShardedIndex.open(tmp_path / "db")
    assert [s["rows"] for s in index.shards] == [256, 44, 200]
    assert torch.equal(_read_all(index)[0], search.prepare_rows(x, "l2"))
    assert list(index.labels) == [str(i) for i in range(500)]  # default labels are global row numbers


def test_writer_refuses_a_mismatched_index_and_bad_rows(tmp_path):
    from esm_b200 import search
    with search.IndexWriter(tmp_path / "db", 320, "cosine", layer=6) as w:
        w.add(_vecs(10, 320, 3))
    for kw, what in ((dict(dim=320, metric="l2", layer=6), "metric"), (dict(dim=480, metric="cosine", layer=6), "dim"),
                     (dict(dim=320, metric="cosine", layer=7), "layer")):
        with pytest.raises(ValueError, match=f"of {what}"):
            search.IndexWriter(tmp_path / "db", **kw)
    w = search.IndexWriter(tmp_path / "db", 320, "cosine", layer=6)
    with pytest.raises(ValueError, match="width 480"):
        w.add(_vecs(3, 480, 4))
    with pytest.raises(ValueError, match="zero row"):
        w.add(torch.zeros(2, 320))
    with pytest.raises(ValueError, match="labels"):
        w.add(_vecs(3, 320, 4), ["a"])
    with pytest.raises(ValueError, match="metric"):
        search.IndexWriter(tmp_path / "other", 320, "dot")
    with pytest.raises(ValueError, match="at least one row"):
        search.IndexWriter(tmp_path / "empty", 320).close()
    assert not (tmp_path / "empty" / "manifest.json").exists()
    (tmp_path / "bad").mkdir()
    (tmp_path / "bad" / "manifest.json").write_text('{"format": "x"}')
    with pytest.raises(ValueError, match="manifest"):
        search.ShardedIndex.open(tmp_path / "bad")
    with pytest.raises(ValueError, match="not a sharded index"):
        search.ShardedIndex.open(tmp_path / "nothing")


def test_one_large_add_is_prepared_a_shard_at_a_time(tmp_path, monkeypatch):
    """A batch of many shards: each prepare_rows call sees at most one shard's rows, each shard is concatenated once,
    and the rows equal the whole batch's prepared rows."""
    from esm_b200 import search
    calls = []
    real = search.prepare_rows
    monkeypatch.setattr(search, "prepare_rows", lambda x, *a, **kw: calls.append(x.shape[0]) or real(x, *a, **kw))
    x = _vecs(1000, 320, 13)
    with search.IndexWriter(tmp_path / "db", 320, "l2", shard_rows=128) as w:
        w.add(x[:50])
        w.add(x[50:])
    assert max(calls) <= 128 and sum(calls) == 1000 and calls[:3] == [50, 78, 128]
    index = search.ShardedIndex.open(tmp_path / "db")
    assert [s["rows"] for s in index.shards] == [128] * 7 + [104]
    rows, beta = _read_all(index)
    assert torch.equal(rows, real(x, "l2")) and torch.equal(-beta, search.squared_norms(real(x, "l2")))


def test_a_refused_add_leaves_the_writer_as_it_was(tmp_path):
    from esm_b200 import search
    x = _vecs(700, 320, 14)
    bad = x.clone()
    bad[650] = 0  # a zero row in the sixth shard-sized slice of the batch
    w = search.IndexWriter(tmp_path / "db", 320, "cosine", shard_rows=100)
    w.add(x[:30])
    with pytest.raises(ValueError, match="zero row"):
        w.add(bad, [f"b{i}" for i in range(700)])
    assert len(w) == 30
    w.add(x[30:])
    w.close()
    index = search.ShardedIndex.open(tmp_path / "db")
    assert torch.equal(_read_all(index)[0], search.prepare_rows(x, "cosine"))
    assert list(index.labels) == [str(i) for i in range(700)]


def test_shards_and_the_manifest_are_fsynced_before_the_manifest_names_them(tmp_path, monkeypatch):
    from esm_b200 import search
    events = []
    real_fsync, real_replace = os.fsync, os.replace
    monkeypatch.setattr(search.os, "fsync", lambda fd: events.append(("fsync", os.readlink(f"/proc/self/fd/{fd}")))
                        or real_fsync(fd))
    monkeypatch.setattr(search.os, "replace", lambda a, b: events.append(("replace", str(b))) or real_replace(a, b))
    with search.IndexWriter(tmp_path / "db", 320, "l2", shard_rows=100) as w:
        w.add(_vecs(150, 320, 15))
    synced = [p for e, p in events if e == "fsync"]
    at = [e for e, _ in events].index("replace")
    for name in ("shard-00000.f16", "shard-00000.norms", "shard-00000.labels.json", "shard-00001.f16"):
        assert any(p.endswith(name) for p in synced[:at]), name
    assert str(tmp_path / "db") in synced[:at] and str(tmp_path / "db") in synced[at:]  # the directory, both sides


def test_a_writer_stopped_before_close_leaves_the_old_index(tmp_path):
    from esm_b200 import search
    x = _vecs(300, 320, 5)
    with search.IndexWriter(tmp_path / "db", 320, shard_rows=100) as w:
        w.add(x[:150])
    before = (tmp_path / "db" / "manifest.json").read_text()
    w = search.IndexWriter(tmp_path / "db", 320, shard_rows=100)
    w.add(x[150:])  # writes shard files, but no manifest
    with pytest.raises(RuntimeError):
        with search.IndexWriter(tmp_path / "db", 320, shard_rows=100) as w2:
            w2.add(x[150:])
            raise RuntimeError("stopped")
    assert (tmp_path / "db" / "manifest.json").read_text() == before
    index = search.ShardedIndex.open(tmp_path / "db")
    assert len(index) == 150 and torch.equal(_read_all(index)[0], search.prepare_rows(x[:150], "cosine"))
    assert not any(f.name.startswith(".manifest") for f in (tmp_path / "db").iterdir())


# ---- chunk planning ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric", ["cosine", "l2"])
@pytest.mark.parametrize("Q,k,D", [(1, 10, 1280), (1000, 128, 320), (8192, 10, 1280), (20_000, 64, 5120)])
def test_chunks_are_whole_tiles_within_the_cap(metric, Q, k, D):
    from esm_b200 import search
    fixed = search._fixed_device_bytes(Q, Q, k, D, metric, 132)
    for cap in (fixed + 2 * 256 * (2 * D + 4), fixed + 7 * 2 * 256 * (2 * D + 4) + 5, 10 ** 9, 80 * 10 ** 9):
        if cap < fixed:
            continue
        rows = search.plan_chunk_rows(Q, Q, k, D, metric, cap, 132)
        assert rows % 256 == 0 and rows >= 256
        assert search.device_bytes(Q, Q, k, D, metric, rows, 132) <= cap
        row = 2 * D + (4 if metric == "l2" else 0)
        assert rows * row <= max(search.MAX_SLOT_BYTES, 256 * row)
        # one more tile would not fit, unless the slot cap stopped it
        more = search.device_bytes(Q, Q, k, D, metric, rows + 256, 132)
        assert more > cap or (rows + 256) * row > search.MAX_SLOT_BYTES
    with pytest.raises(ValueError, match="leaves no room"):
        search.plan_chunk_rows(Q, Q, k, D, metric, fixed + 100, 132)


def _launched_batches(Q, block):
    """The query-batch sizes ShardedIndex._stream launches for Q queries held `block` rows at a time."""
    from esm_b200 import search
    for a0 in range(0, Q, block):
        a1 = min(Q, a0 + block)
        for b0 in range(0, a1 - a0, search.QUERY_BATCH):
            yield min(a1 - a0, b0 + search.QUERY_BATCH) - b0


@pytest.mark.parametrize("num_sms", [78, 114, 132, 144])
@pytest.mark.parametrize("query_batch", [8192, 1024])
def test_the_scratch_covers_every_batch_a_call_launches(num_sms, query_batch, monkeypatch):
    """Splits times batch size is not monotone in the batch size: a short last batch can need more scratch than a
    full one (Q = 10,533 on 114 SMs: 8,192 queries at 2 stripes, then 2,341 at 7). Every batch a search() or a
    blocked search_all() launches, at every chunk length, must fit the scratch and the budget the call plans."""
    from esm_b200 import search
    monkeypatch.setattr(search, "QUERY_BATCH", query_batch)
    qb = query_batch
    qs = sorted({10_533, 1, 63, 64, 65} | {m * qb + d for m in range(1, 4) for d in (-2049, -1, 0, 1, 37, 2341, 3001)
                                            if m * qb + d > 0} | set(range(1, 3 * qb, 97)))
    for Q in qs:
        for block in {Q, 64, 1856, qb, 3 * qb // 2}:
            if block > Q:
                continue
            need = search.scratch_bytes(block, Q, 128, num_sms)
            fixed = search._fixed_device_bytes(block, Q, 128, 1280, "cosine", num_sms)
            for b in set(_launched_batches(Q, block)):
                for n in (256, 3 * 256 + 5, 10**6):
                    got = search.choose_splits(b, n, num_sms) * b * 128 * 8
                    assert got <= need <= fixed, (Q, block, b, n)
    # the case from the example, with the library's own size function
    from esm_b200 import _lib
    lib = _lib.load()
    nb = ctypes.c_size_t(0)
    monkeypatch.setattr(search, "QUERY_BATCH", 8192)
    assert lib.esmb200_knn_scratch_bytes(2341, 10, search.choose_splits(2341, 10**6, 114), ctypes.byref(nb)) == 0
    assert nb.value > lib_bytes(lib, 8192, 10, search.choose_splits(8192, 10**6, 114))
    assert search.scratch_bytes(10_533, 10_533, 10, 114) >= nb.value


def lib_bytes(lib, Q, k, splits):
    nb = ctypes.c_size_t(0)
    assert lib.esmb200_knn_scratch_bytes(Q, k, splits, ctypes.byref(nb)) == 0
    return nb.value


# ---- the command line --------------------------------------------------------------------------------------------------
def test_cli_parses_the_new_forms():
    from esm_b200 import search_cli
    p = search_cli.create_parser()
    a = p.parse_args(["build", "ex", "--layer", "33", "--out", "db"])
    assert not a.append and str(a.out) == "db" and not search_cli._is_file_index(a.out)
    a = p.parse_args(["build", "ex", "--layer", "33", "--out", "db", "--append", "--shard-rows", "1000"])
    assert a.append and a.shard_rows == 1000
    assert search_cli._is_file_index(p.parse_args(["build", "ex", "--layer", "3", "--out", "x/db.pt"]).out)
    a = p.parse_args(["query", "db", "--queries", "q", "--k", "7", "--out", "h.tsv"])
    assert str(a.index) == "db" and a.k == 7


def _write(root, label, vec, layer):
    path = root / f"{label}.pt"
    path.parent.mkdir(parents=True, exist_ok=True)
    torch.save({"label": label, "mean_representations": {layer: vec.clone()}}, path)


def test_cli_build_writes_rows_in_label_order_and_appends(tmp_path, monkeypatch):
    from esm_b200 import search, search_cli
    monkeypatch.setattr(search_cli, "BUILD_BATCH", 7)
    g = torch.Generator().manual_seed(6)
    labels = [f"fam{i % 3}/p{(i * 37) % 50:03d}" for i in range(50)]
    vecs = {l: torch.randn(320, generator=g) for l in labels}
    for l in labels:
        _write(tmp_path / "ex", l, vecs[l], 33)
    p = search_cli.create_parser()
    n = search_cli.run(p.parse_args(["build", str(tmp_path / "ex"), "--layer", "33", "--metric", "l2", "--out",
                                     str(tmp_path / "db"), "--shard-rows", "16"]))
    assert n == 50
    index = search.ShardedIndex.open(tmp_path / "db")
    ref = search.EmbeddingIndex.from_extract_dir(tmp_path / "ex", 33, "l2")
    assert list(index.labels) == ref.labels and torch.equal(_read_all(index)[0], ref.rows)
    with pytest.raises(ValueError, match="--append"):
        search_cli.run(p.parse_args(["build", str(tmp_path / "ex"), "--layer", "33", "--metric", "l2", "--out",
                                     str(tmp_path / "db")]))
    with pytest.raises(ValueError, match="metric"):
        search_cli.run(p.parse_args(["build", str(tmp_path / "ex"), "--layer", "33", "--out", str(tmp_path / "db"),
                                     "--append"]))
    with pytest.raises(ValueError, match="existing"):
        search_cli.run(p.parse_args(["build", str(tmp_path / "ex"), "--layer", "33", "--out", str(tmp_path / "no"),
                                     "--append"]))
    with pytest.raises(ValueError, match="not to a .pt"):
        search_cli.run(p.parse_args(["build", str(tmp_path / "ex"), "--layer", "33", "--out", str(tmp_path / "a.pt"),
                                     "--append"]))
    search_cli.run(p.parse_args(["build", str(tmp_path / "ex"), "--layer", "33", "--metric", "l2", "--out",
                                 str(tmp_path / "db"), "--append"]))
    index = search.ShardedIndex.open(tmp_path / "db")
    assert len(index) == 100 and list(index.labels) == ref.labels * 2


def test_cli_query_on_a_directory_refuses_before_any_work(tmp_path):
    from esm_b200 import search, search_cli
    g = torch.Generator().manual_seed(12)
    with search.IndexWriter(tmp_path / "db", 320, layer=33) as w:
        w.add(torch.randn(10, 320, generator=g))
    _write(tmp_path / "q1", "x", torch.randn(480, generator=g), 33)
    p = search_cli.create_parser()
    with pytest.raises(ValueError, match="width 480"):
        search_cli.run(p.parse_args(["query", str(tmp_path / "db"), "--queries", str(tmp_path / "q1"),
                                     "--out", str(tmp_path / "h.tsv")]))
    with pytest.raises(ValueError, match=r"k must be in \[1, 9\]"):
        search_cli.run(p.parse_args(["query", str(tmp_path / "db"), "--all", "--k", "10",
                                     "--out", str(tmp_path / "h.tsv")]))
    assert not (tmp_path / "h.tsv").exists()


# ---- Python refusals ---------------------------------------------------------------------------------------------------
def test_sharded_search_refuses_bad_arguments_before_the_device(tmp_path):
    from esm_b200 import search
    x = _vecs(20, 64, 10)
    with search.IndexWriter(tmp_path / "db", 64) as w:
        w.add(x)
    index = search.ShardedIndex.open(tmp_path / "db")
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


@pytest.mark.skipif(torch.cuda.is_available(), reason="the refusal for a machine without a CUDA device")
def test_sharded_search_needs_a_cuda_device(tmp_path):
    from esm_b200 import search
    with search.IndexWriter(tmp_path / "db", 64) as w:
        w.add(_vecs(20, 64, 11))
    index = search.ShardedIndex.open(tmp_path / "db")
    with pytest.raises(ValueError, match="CUDA device"):
        index.search(_vecs(2, 64, 12), k=3)
    with pytest.raises(ValueError, match="CUDA device"):
        index.search_all(k=3)


# ---- the C ABI ---------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_and_exported():
    from esm_b200 import _lib
    text = open(os.path.join(os.path.dirname(HERE), "include", "esmb200.h")).read()
    lib = _lib.load()
    for name in ("esmb200_knn_search_accumulate", "esmb200_knn_decode"):
        assert re.search(rf"\b{name}\s*\(", text) and name in _lib.EXPORTS and hasattr(lib, name)
    assert lib.esmb200_abi_version() == 4


# Placeholder pointers, which a refused call never dereferences; only where no CUDA device is present (the pattern of
# tests/test_search_host.py). tests/test_gpu_search_shards.py repeats every refusal with real buffers.
_FAKE = 4096
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="placeholder pointers: only where nothing can launch")
ACC_ARGS = dict(queries=_FAKE, q_ld=320, Q=8, base=_FAKE, b_ld=320, n=300, row0=1000, D=320, beta=None, alpha=1.0,
                self_offset=-1, k=10, splits=2, scratch=_FAKE, scratch_bytes=1 << 20, keys=_FAKE)
ACC_REFUSALS = [
    ({"queries": None}, "null"), ({"base": None}, "null"), ({"scratch": None}, "null"), ({"keys": None}, "null"),
    ({"k": 0}, "1 <= k <= 128"), ({"k": 129}, "1 <= k <= 128"),
    ({"D": 100}, "D % 64"), ({"D": 0}, "D % 64"),
    ({"q_ld": 300}, "q_ld"), ({"b_ld": 324}, "b_ld"),
    ({"queries": _FAKE + 8}, "16-byte aligned"), ({"base": _FAKE + 2}, "16-byte aligned"),
    ({"keys": _FAKE + 4}, "8-byte aligned"),
    ({"splits": 0}, "splits"), ({"splits": 1025}, "splits"),
    ({"scratch_bytes": 8 * 2 * 10 * 8 - 1}, "scratch smaller"),
    ({"Q": -1}, "Q >= 0"), ({"n": 0}, "n >= 1"), ({"row0": -1}, "row0 >= 0"),
    ({"row0": (1 << 31) - 300}, "row0 + n < 2^31"), ({"n": 1 << 31, "row0": 0}, "row0 + n < 2^31"),
]
DEC_ARGS = dict(keys=_FAKE, Q=8, k=10, out_scores=_FAKE, out_idx=_FAKE)
DEC_REFUSALS = [({"keys": None}, "null"), ({"out_scores": None}, "null"), ({"out_idx": None}, "null"),
                ({"keys": _FAKE + 4}, "8-byte aligned"), ({"out_scores": _FAKE + 2}, "4-byte aligned out_scores"),
                ({"out_idx": _FAKE + 4}, "8-byte aligned out_idx"), ({"Q": -1}, "Q >= 0"),
                ({"k": 0}, "1 <= k <= 128"), ({"k": 129}, "1 <= k <= 128")]


def _ids(v):
    return v if isinstance(v, str) else "-".join(v) if isinstance(v, dict) else ""


@no_device
@pytest.mark.parametrize("over,msg", ACC_REFUSALS, ids=_ids)
def test_knn_search_accumulate_refuses_bad_arguments(over, msg):
    from esm_b200 import _lib
    lib = _lib.load()
    kw = dict(ACC_ARGS, **over)
    before = lib.esmb200_launch_count()
    rc = lib.esmb200_knn_search_accumulate(*kw.values(), None)
    assert rc == -1 and msg in lib.esmb200_last_error().decode(), lib.esmb200_last_error()
    assert lib.esmb200_launch_count() == before


@no_device
@pytest.mark.parametrize("over,msg", DEC_REFUSALS, ids=_ids)
def test_knn_decode_refuses_bad_arguments(over, msg):
    from esm_b200 import _lib
    lib = _lib.load()
    kw = dict(DEC_ARGS, **over)
    before = lib.esmb200_launch_count()
    rc = lib.esmb200_knn_decode(*kw.values(), None)
    assert rc == -1 and msg in lib.esmb200_last_error().decode(), lib.esmb200_last_error()
    assert lib.esmb200_launch_count() == before
