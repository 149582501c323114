"""CPU: range search (esm_b200.search range_search / esmb200_knn_range) without a GPU. The new symbols, the C-ABI
refusals with placeholder pointers, the Python refusals, the l2 threshold bisection checked by bit pattern, the CSR
restatement and max_hits truncation, the batch and overflow planning, and the CLI's range command and refusals."""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

from range_refs import csr_of_hits

HERE = os.path.dirname(os.path.abspath(__file__))
NEW = ("esmb200_knn_range", "esmb200_knn_range_finish_scratch_bytes", "esmb200_knn_range_finish")


def test_symbols_declared_exported_and_abi_4():
    from esm_b200 import _lib
    header = open(os.path.join(HERE, "..", "include", "esmb200.h")).read()
    assert re.search(r"#define ESMB200_ABI_VERSION 4\b", header)
    lib = _lib.load()
    assert lib.esmb200_abi_version() == 4
    for name in NEW:
        assert re.search(rf"\bint {name}\(", header), name
        assert name in _lib.EXPORTS
        assert hasattr(lib, name)


# ---- C-ABI refusals (all before any launch, so placeholder pointers do) --------------------------------------------
def _range_args(**over):
    kw = dict(queries=256, q_ld=128, Q=10, base=512, b_ld=128, n=1000, row0=0, D=128, beta=None, alpha=1.0,
              self_offset=-1, tau=1024, splits=4, hit_keys=2048, hit_rows=4096, hit_cap=100, hit_counts=8192,
              hit_total=16384)
    kw.update(over)
    return kw


@pytest.mark.parametrize("over,msg", [
    (dict(Q=-1), "Q >= 0"), (dict(n=0), "n >= 1"), (dict(row0=-1), "row0 >= 0"),
    (dict(row0=(1 << 31) - 10, n=10), "row0 + n < 2^31"), (dict(D=96), "D % 64"), (dict(q_ld=100), "q_ld"),
    (dict(b_ld=64), "b_ld"), (dict(splits=0), "splits"), (dict(splits=1025), "splits"),
    (dict(hit_cap=-1), "hit_cap"), (dict(hit_cap=1 << 31), "hit_cap"), (dict(tau=None), "null"),
    (dict(hit_counts=None), "null"), (dict(hit_total=None), "null"), (dict(hit_keys=None), "null"),
    (dict(hit_rows=None), "null"), (dict(queries=8), "16-byte"), (dict(base=24), "16-byte"),
    (dict(tau=1026), "aligned"), (dict(hit_keys=2052), "aligned"), (dict(hit_rows=4098), "aligned"),
    (dict(hit_counts=8196), "aligned"), (dict(hit_total=16388), "aligned"), (dict(beta=2), "aligned"),
])
def test_knn_range_refusals(over, msg):
    from esm_b200 import _lib
    lib = _lib.load()
    rc = lib.esmb200_knn_range(*_range_args(**over).values(), None)
    assert rc == -1 and msg in lib.esmb200_last_error().decode(), lib.esmb200_last_error()


def test_knn_range_counting_only_takes_null_buffers():
    """hit_cap 0 with NULL hit buffers is a counting call: it passes every check (Q == 0 then launches nothing)."""
    from esm_b200 import _lib
    lib = _lib.load()
    assert lib.esmb200_knn_range(*_range_args(Q=0, hit_cap=0, hit_keys=None, hit_rows=None).values(), None) == 0


def _finish_args(**over):
    kw = dict(keys=256, rows=512, nnz=100, counts=1024, Q=10, max_hits=-1, scratch=2048, scratch_bytes=88,
              lims=4096, scores=8192, idx=16384)
    kw.update(over)
    return kw


@pytest.mark.parametrize("over,msg", [
    (dict(Q=-1), "Q >= 0"), (dict(nnz=-1), "nnz"), (dict(nnz=1 << 31), "nnz < 2^31"), (dict(max_hits=0), "max_hits"),
    (dict(max_hits=-2), "max_hits"), (dict(counts=None), "null"), (dict(scratch=None), "null"),
    (dict(lims=None), "null"), (dict(keys=None), "null"), (dict(rows=None), "null"), (dict(scores=None), "null"),
    (dict(idx=None), "null"), (dict(keys=260), "aligned"), (dict(rows=514), "aligned"), (dict(counts=1028), "aligned"),
    (dict(scratch=2052), "aligned"), (dict(lims=4100), "aligned"), (dict(scores=8194), "aligned"),
    (dict(idx=16388), "aligned"), (dict(scratch_bytes=87), "scratch smaller"),
])
def test_knn_range_finish_refusals(over, msg):
    from esm_b200 import _lib
    lib = _lib.load()
    rc = lib.esmb200_knn_range_finish(*_finish_args(**over).values(), None)
    assert rc == -1 and msg in lib.esmb200_last_error().decode(), lib.esmb200_last_error()


def test_finish_scratch_bytes():
    from esm_b200 import _lib
    lib = _lib.load()
    out = ctypes.c_size_t(0)
    for Q in (0, 1, 8192):
        assert lib.esmb200_knn_range_finish_scratch_bytes(Q, ctypes.byref(out)) == 0 and out.value == (Q + 1) * 8
    assert lib.esmb200_knn_range_finish_scratch_bytes(-1, ctypes.byref(out)) == -1
    assert lib.esmb200_knn_range_finish_scratch_bytes(1, None) == -1


# ---- Python refusals ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("metric,kw,msg", [
    ("cosine", {}, "exactly one threshold"),
    ("cosine", dict(min_score=0.5, max_distance=1.0), "exactly one threshold"),
    ("cosine", dict(max_distance=1.0), "takes min_score"),
    ("l2", dict(min_score=0.5), "takes max_distance"),
    ("cosine", dict(min_score=float("nan")), "NaN"),
    ("l2", dict(max_distance=float("nan")), "NaN"),
    ("l2", dict(max_distance=-1e-30), ">= 0"),
    ("cosine", dict(min_score="0.5"), "real number"),
    ("cosine", dict(min_score=True), "real number"),
    ("cosine", dict(min_score=0.5, max_hits=0), "max_hits"),
    ("cosine", dict(min_score=0.5, max_hits=2.0), "max_hits"),
])
def test_range_argument_refusals(metric, kw, msg):
    from esm_b200 import search
    index = search.EmbeddingIndex(torch.randn(5, 64), metric=metric)  # on the CPU: the checks come first
    with pytest.raises(ValueError, match=msg):
        index.range_search(torch.randn(2, 64), **kw)
    with pytest.raises(ValueError, match=msg):
        index.range_search_all(**kw)


def test_range_search_needs_a_gpu_index():
    from esm_b200 import search
    index = search.EmbeddingIndex(torch.randn(5, 64))
    with pytest.raises(ValueError, match="on the CPU"):
        index.range_search(torch.randn(2, 64), min_score=0.5)


def test_threshold_rounding_to_fp32():
    from esm_b200 import search
    np.seterr(over="ignore")
    for x in (0.1, -0.1, 0.9, 1e-40, -1e-40, 1e300, -1e300, 3.4028235e38, float("inf"), float("-inf"), 0.0, -0.0):
        up, dn = search.fp32_at_or_above(x), search.fp32_at_or_below(x)
        assert up >= x and dn <= x and float(np.float32(up)) == up and float(np.float32(dn)) == dn
        if math.isfinite(up) and up > x:
            assert float(np.nextafter(np.float32(up), np.float32(-np.inf))) < x
        if math.isfinite(dn) and dn < x:
            assert float(np.nextafter(np.float32(dn), np.float32(np.inf))) > x


# ---- the l2 threshold, by bit pattern ----------------------------------------------------------------------------------
def _neighbourhood(t: float, w: int) -> torch.Tensor:
    """The 2w + 1 fp32 values around t (by ordered bit pattern), within [-inf, +inf]."""
    from esm_b200 import search
    o = torch.tensor([t], dtype=torch.float32).view(torch.int32).long()
    o = torch.where(o >= 0, o, -(o & 0x7FFFFFFF) - 1)
    r = torch.arange(-w, w + 1) + o
    r = r.clamp(search._ORD_NEG_INF, search._ORD_POS_INF).unique()
    return search._f32_of_ordinal(r)


@pytest.mark.parametrize("qn,r", [
    (1.0, 0.5), (1.0, 0.0), (1.0, float("inf")), (1.0, 1e-3), (3.25, 1.75), (0.0, 0.0), (0.0, 1.0), (1e-30, 1e-20),
    (1e30, 1e10), (4096.0, 64.0), (2.0, 1.0), (123.456, 3.0), (1.0, 1.0), (7.0, 1e-45), (65504.0, 1e38),
])
def test_l2_threshold_is_exact_by_bit_pattern(qn, r):
    """s >= tau <=> distance(s) <= r over every fp32 s near tau, near |q|^2 - r^2 and near |q|^2 (where |q|^2 - s
    crosses 0)."""
    from esm_b200 import search
    qn32 = torch.tensor([qn], dtype=torch.float32)
    tau = search.l2_thresholds(qn32, r)
    t = float(tau[0])
    assert not (t == 0 and math.copysign(1, t) < 0), "tau is -0"
    r32 = search.fp32_at_or_below(r)
    pts = [t, float(qn32[0]), float(qn32[0]) - min(r32 * r32, 3e38), 0.0]
    s = torch.cat([_neighbourhood(p, 3000) for p in pts if math.isfinite(p)] + [_neighbourhood(t, 3000)]).unique()
    d = search.l2_distance(qn32.expand_as(s), s)
    assert torch.equal(s >= tau, d.double() <= r), f"tau {t!r} disagrees with the distance test"
    if r == float("inf"):
        assert t == float("-inf")


def test_l2_threshold_many_pairs():
    from esm_b200 import search
    g = torch.Generator().manual_seed(3)
    qn = (torch.rand(400, generator=g) * 10).pow(3).float()
    for r in (0.0, 0.3, 1.0, 2.5, 30.0, float("inf")):
        tau = search.l2_thresholds(qn, r)
        ok = search.l2_distance(qn, tau).double() <= r
        assert bool(ok.all())
        below = torch.from_numpy(np.nextafter(tau.numpy(), np.float32(-np.inf)))
        finite = torch.isfinite(tau)
        assert not bool((search.l2_distance(qn, below).double() <= r)[finite].any()), "tau is not the smallest qualifying s"


def test_cosine_thresholds_normalise_minus_zero():
    from esm_b200 import search
    tau = search.range_thresholds("cosine", None, 3, -0.0, None, "cpu")
    assert torch.equal(tau.view(torch.int32), torch.zeros(3, dtype=torch.int32))
    assert float(search.range_thresholds("cosine", None, 1, 0.1, None, "cpu")[0]) == search.fp32_at_or_above(0.1)


# ---- CSR restatement and planning ---------------------------------------------------------------------------------------
def test_csr_restatement_ignores_append_order_and_truncates():
    g = torch.Generator().manual_seed(0)
    Q, nnz = 7, 300
    b = torch.randperm(10 ** 6, generator=g)[:nnz].long() - (1 << 62)  # distinct keys
    rows = torch.randint(0, Q - 1, (nnz,), generator=g)  # the last query has no hit
    lims, keys = csr_of_hits(b, rows, Q)
    perm = torch.randperm(nnz, generator=g)
    lims2, keys2 = csr_of_hits(b[perm], rows[perm], Q)
    assert torch.equal(lims, lims2) and torch.equal(keys, keys2)
    assert lims[-1] == nnz and lims[-1] == lims[-2]
    for M in (1, 5, 1000):
        lm, km = csr_of_hits(b, rows, Q, M)
        for q in range(Q):
            assert torch.equal(km[lm[q]:lm[q + 1]], keys[lims[q]:lims[q + 1]][:M])
            assert lm[q + 1] - lm[q] == min(M, lims[q + 1] - lims[q])


def test_plan_range_reruns():
    from esm_b200 import search
    assert search.plan_range_reruns([3, 4, 2, 5, 0, 1], 7, "min_score 0.5") == [(0, 2), (2, 5), (5, 6)]
    assert search.plan_range_reruns([0, 0, 0], 1, "t") == [(0, 3)]
    assert search.plan_range_reruns([7], 7, "t") == [(0, 1)]
    for counts, cap in (([5] * 10, 12), ([1, 9, 3, 3, 3, 8], 9), ([0] * 4 + [4], 4)):
        groups = search.plan_range_reruns(counts, cap, "t")
        assert [c for a, b in groups for c in range(a, b)] == list(range(len(counts)))
        assert all(sum(counts[a:b]) <= cap for a, b in groups)
    with pytest.raises(ValueError, match=r"query 12 has 9 hits at min_score 0\.25"):
        search.plan_range_reruns([1, 9], 8, "min_score 0.25", q_base=11)


def test_plan_range_stream():
    from esm_b200 import search
    D = 1280
    row = search._row_bytes(D, "cosine")
    block, chunk, hit_cap = search.plan_range_stream(10 ** 6, 100, D, "cosine", 8 << 30)
    assert block == 100 and hit_cap == search.range_hit_cap() and chunk % search.TILE == 0
    assert chunk * row <= search.MAX_SLOT_BYTES
    # a small budget: a quarter for hits, the block within half, the ring in the rest
    cap = 64 << 20
    block, chunk, hit_cap = search.plan_range_stream(10 ** 6, 10 ** 6, D, "l2", cap)
    assert block % 64 == 0 and 64 <= block < 10 ** 6 and hit_cap == cap // 4 // search.HIT_BYTES
    per_query = D * 2 + 16
    used = block * per_query + hit_cap * search.HIT_BYTES + search.RING_SLOTS * chunk * search._row_bytes(D, "l2")
    assert used <= cap
    assert search.plan_range_stream(1000, 5, D, "cosine", 8 << 30)[1] == 1024  # no chunk past the database
    with pytest.raises(ValueError, match="max_device_bytes"):
        search.plan_range_stream(10 ** 6, 10 ** 6, D, "cosine", 1 << 20)


# ---- CLI -------------------------------------------------------------------------------------------------------------------
def test_cli_parses_range():
    from esm_b200 import search_cli
    p = search_cli.create_parser()
    a = p.parse_args(["range", "db.pt", "--all", "--min-score", "0.9", "--max-hits", "500", "--out", "h.tsv"])
    assert a.command == "range" and a.all and a.min_score == 0.9 and a.max_hits == 500 and a.max_distance is None
    a = p.parse_args(["range", "db/", "--queries", "q/", "--max-distance", "2.5", "--out", "h.tsv"])
    assert a.max_distance == 2.5 and a.min_score is None
    for bad in (["range", "db.pt", "--all", "--min-score", "1", "--max-distance", "1", "--out", "h"],
                ["range", "db.pt", "--all", "--out", "h"],
                ["range", "db.pt", "--min-score", "1", "--out", "h"]):
        with pytest.raises(SystemExit):
            p.parse_args(bad)
    q = p.parse_args(["query", "db.pt", "--all", "--out", "h.tsv"])
    assert q.k == 10  # the query command is unchanged


def _run(argv):
    from esm_b200 import search_cli
    return search_cli.run(search_cli.create_parser().parse_args(argv))


def test_cli_range_refusals(tmp_path):
    from esm_b200 import search
    x = torch.randn(20, 64, generator=torch.Generator().manual_seed(0))
    search.EmbeddingIndex(x, metric="cosine", layer=3).save(tmp_path / "cos.pt")
    search.EmbeddingIndex(x, metric="l2", layer=3).save(tmp_path / "l2.pt")
    out = str(tmp_path / "h.tsv")
    with pytest.raises(ValueError, match="takes min_score"):
        _run(["range", str(tmp_path / "cos.pt"), "--all", "--max-distance", "1", "--out", out])
    with pytest.raises(ValueError, match="takes max_distance"):
        _run(["range", str(tmp_path / "l2.pt"), "--all", "--min-score", "0.5", "--out", out])
    with pytest.raises(ValueError, match="NaN"):
        _run(["range", str(tmp_path / "cos.pt"), "--all", "--min-score", "nan", "--out", out])
    with pytest.raises(ValueError, match="max_hits"):
        _run(["range", str(tmp_path / "cos.pt"), "--all", "--min-score", "0.5", "--max-hits", "0", "--out", out])
    rows = search.prepare_rows(x, "cosine")
    ivf = search.IVFIndex._from_parts(rows, torch.arange(20), torch.tensor([0, 20]), rows[:1], 64,
                                      [str(i) for i in range(20)], "cosine", 3, {"nlist": 1})
    ivf.save(tmp_path / "ivf.pt")
    with pytest.raises(ValueError, match="IVF index"):
        _run(["range", str(tmp_path / "ivf.pt"), "--all", "--min-score", "0.5", "--out", out])
    assert not os.path.exists(out)


def test_write_hits_from_csr(tmp_path):
    from esm_b200 import search_cli
    lims = torch.tensor([0, 2, 2, 3])
    scores, idx = torch.tensor([0.9, 0.5, 0.7]), torch.tensor([4, 1, 0])
    n = search_cli.write_hits(tmp_path / "h.tsv", ["a", "b", "c"], ["t0", "t1", "t2", "t3", "t4"],
                              search_cli.csr_rows(lims, scores), search_cli.csr_rows(lims, idx))
    assert n == 3
    assert (tmp_path / "h.tsv").read_text().splitlines() == [
        "query\trank\ttarget\tscore", "a\t1\tt4\t0.9", "a\t2\tt1\t0.5", "c\t1\tt0\t0.7"]
