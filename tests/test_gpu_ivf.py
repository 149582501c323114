"""GPU: the inverted-file index (esm_b200.search.IVFIndex, esmb200_ivf_search, esmb200_kmeans_means). With every list
probed it must equal EmbeddingIndex bit for bit; with fewer, each query must get the exact search over the rows of
its probed lists, bit for bit; k-means means must equal the exact CPU reference, and builds must be deterministic."""
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import ivf_refs  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _designed(metric, N=3000, E=320, nlist=8, seed=0):
    """An EmbeddingIndex and an IVFIndex of the same rows with hand-made lists: list 0 holds half the rows (several
    stripes of one tile), list 3 is empty, list 5 holds one row, and five rows appear twice, in different lists."""
    from esm_b200 import search
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, E, generator=g)
    x[N - 5:] = x[:5]  # duplicates: equal scores, ties decided by the original index
    exact = search.EmbeddingIndex(x, metric=metric, layer=33).to(DEV)
    a = torch.randint(0, nlist, (N,), generator=g)
    a[a == 3] = 4
    a[a == 5] = 6
    a[7] = 5
    a[torch.randperm(N, generator=g)[:N // 2]] = 0
    a[7] = 5
    a[:5] = 1
    a[N - 5:] = 2
    ids = torch.sort(a, stable=True).indices
    offsets = torch.zeros(nlist + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.bincount(a, minlength=nlist), 0)
    cent = search.prepare_rows(torch.randn(nlist, E, generator=g), metric)
    ivf = search.IVFIndex._from_parts(exact.rows[ids.to(DEV)], ids.to(DEV), offsets.to(DEV), cent.to(DEV), E,
                                      exact.labels, metric, 33, {"nlist": nlist})
    return exact, ivf


@pytest.mark.parametrize("metric", ["cosine", "l2"])
@pytest.mark.parametrize("k", [1, 10, 128])
def test_every_list_equals_the_exact_index(metric, k):
    exact, ivf = _designed(metric)
    offs = ivf.offsets.tolist()
    assert offs[4] == offs[3] and offs[6] - offs[5] == 1 and offs[1] - offs[0] >= 1500
    g = torch.Generator().manual_seed(5)
    for Q in (1, 63, 64, 65, 300):
        q = torch.randn(Q, 320, generator=g)
        q[0] = exact.rows[3, :320].float().cpu()  # a query on a duplicated row: two equal best scores
        a, b = exact.search(q, k), ivf.search(q, k, nprobe=ivf.nlist)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), (Q, k)
    a, b = exact.search_all(k), ivf.search_all(k, nprobe=ivf.nlist)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_every_list_past_one_query_batch(monkeypatch):
    from esm_b200 import search
    exact, ivf = _designed("cosine")
    n = search.ivf_query_batch(ivf.nlist, ivf.nlist, len(ivf), 320, 10, cap=search.ivf_scratch_bytes(
        100, ivf.nlist, ivf.nlist, len(ivf), 320, 10))
    monkeypatch.setattr(search, "IVF_SCRATCH_CAP", search.ivf_scratch_bytes(100, ivf.nlist, ivf.nlist, len(ivf), 320, 10))
    assert n < 1000
    a, b = exact.search_all(10), ivf.search_all(10, nprobe=ivf.nlist)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def _check_probed(ivf, q, k, nprobe, self_rows=False):
    """Each query's result against the exact kernel over exactly the rows of its probed lists."""
    from esm_b200 import search
    probes = ivf.probes(q, nprobe)
    alpha = 2.0 if ivf.metric == "l2" else 1.0
    self_ids = torch.arange(q.shape[0], device=DEV) if self_rows else None
    s, i = search.ivf_search(q, ivf.rows, ivf.ids, ivf.offsets, k, ivf._beta, alpha, probes, self_ids)
    ids_cpu = ivf.ids.cpu()
    for r in range(q.shape[0]):
        pos = ivf_refs.probed_rows(ids_cpu, ivf.offsets.cpu(), probes[r].tolist())
        rs, ri = ivf_refs.topk_over(search, q[r:r + 1], ivf.rows, ids_cpu, ivf._beta, alpha, pos, k,
                                    r if self_rows else -1)
        assert torch.equal(ri, i[r].cpu()), r
        assert torch.equal(rs, s[r].cpu()) or (torch.isnan(rs) == torch.isnan(s[r].cpu())).all() and \
            torch.equal(rs[~torch.isnan(rs)], s[r].cpu()[~torch.isnan(rs)]), r
    return probes, s, i


@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_probed_lists_give_the_exact_search_over_their_rows(metric):
    from esm_b200 import search
    exact, ivf = _designed(metric)
    q = search.prepare_rows(torch.randn(70, 320, generator=torch.Generator().manual_seed(6)), metric).to(DEV)
    for nprobe, k in ((1, 10), (3, 128), (7, 5)):
        probes, s, i = _check_probed(ivf, q, k, nprobe)
        # the probed lists are the top nprobe centroids (float64 scores, with room for fp16 rounding)
        c = ivf.centroids.double()
        cs = 2 * q.double() @ c.T - c.pow(2).sum(1)[None] if metric == "l2" else q.double() @ c.T
        got = cs.gather(1, probes.long())
        rest = cs.scatter(1, probes.long(), float("-inf"))
        assert bool((got.min(1).values >= rest.max(1).values - 1e-2).all())
        assert bool((got[:, :-1] >= got[:, 1:] - 1e-2).all())
        assert len({tuple(sorted(r)) for r in probes.tolist()}) > 1
    # search_all leaves out each row's own original index
    qa = ivf.rows[ivf._pos[:70]]
    _check_probed(ivf, qa, 10, 2, self_rows=True)


def test_probed_stripes_of_several_tiles_at_unaligned_list_offsets():
    from esm_b200 import search
    N, nlist = 40000, 8
    exact, ivf = _designed("l2", N=N, nlist=nlist)
    T = -(-(-(-N // 256) + nlist) // 64)  # tiles per stripe of a probed search (include/esmb200.h)
    offs = ivf.offsets.tolist()
    assert T >= 3 and offs[1] - offs[0] > 4 * 256 * T  # list 0 runs as several multi-tile stripes
    assert any(o % 256 for o in offs[1:-1])
    q = search.prepare_rows(torch.randn(40, 320, generator=torch.Generator().manual_seed(14)), "l2").to(DEV)
    for nprobe, k in ((2, 10), (5, 128)):
        _check_probed(ivf, q, k, nprobe)
    # a probe set that starts with list 0 on every query, so every stripe of it is scanned
    probes = torch.stack([torch.zeros(40, dtype=torch.int32, device=DEV), ivf.probes(q, 1)[:, 0]], 1)
    s, i = search.ivf_search(q, ivf.rows, ivf.ids, ivf.offsets, 20, ivf._beta, 2.0, probes)
    for r in range(40):
        pos = ivf_refs.probed_rows(ivf.ids.cpu(), ivf.offsets.cpu(), probes[r].tolist())
        rs, ri = ivf_refs.topk_over(search, q[r:r + 1], ivf.rows, ivf.ids.cpu(), ivf._beta, 2.0, pos, 20)
        assert torch.equal(ri, i[r].cpu()) and torch.equal(rs, s[r].cpu()), r


def test_a_repeated_probe_scans_its_list_once():
    from esm_b200 import search
    exact, ivf = _designed("cosine")
    q = search.prepare_rows(torch.randn(200, 320, generator=torch.Generator().manual_seed(15)), "cosine").to(DEV)
    once = torch.tensor([[0, 2, -1, 1]], dtype=torch.int32, device=DEV).repeat(200, 1)
    twice = torch.tensor([[0, 2, 0, 1]], dtype=torch.int32, device=DEV).repeat(200, 1)
    allsame = torch.zeros((200, 4), dtype=torch.int32, device=DEV)
    a = search.ivf_search(q, ivf.rows, ivf.ids, ivf.offsets, 50, None, 1.0, once)
    b = search.ivf_search(q, ivf.rows, ivf.ids, ivf.offsets, 50, None, 1.0, twice)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    c = search.ivf_search(q, ivf.rows, ivf.ids, ivf.offsets, 50, None, 1.0, allsame)
    d = search.ivf_search(q, ivf.rows, ivf.ids, ivf.offsets, 50, None, 1.0, allsame[:, :1].contiguous())
    assert torch.equal(c[0], d[0]) and torch.equal(c[1], d[1])
    for row in c[1].tolist():
        assert len(set(row)) == len(row)


def test_short_probed_lists_leave_nan_and_minus_one():
    from esm_b200 import search
    exact, ivf = _designed("cosine")
    q = search.prepare_rows(torch.randn(64, 320, generator=torch.Generator().manual_seed(7)), "cosine").to(DEV)
    probes = torch.full((64, 2), 5, dtype=torch.int32, device=DEV)  # the one-row list, and the empty list
    probes[:, 1] = 3
    s, i = search.ivf_search(q, ivf.rows, ivf.ids, ivf.offsets, 4, None, 1.0, probes)
    assert (i[:, 0] == 7).all() and (i[:, 1:] == -1).all() and torch.isnan(s[:, 1:]).all()
    assert not torch.isnan(s[:, 0]).any()
    probes[:, 0] = 3
    s, i = search.ivf_search(q, ivf.rows, ivf.ids, ivf.offsets, 4, None, 1.0, probes)
    assert (i == -1).all() and torch.isnan(s).all()


def test_a_query_does_not_depend_on_its_batch(monkeypatch):
    from esm_b200 import search
    exact, ivf = _designed("l2")
    q = torch.randn(200, 320, generator=torch.Generator().manual_seed(8))
    whole = ivf.search(q, 10, nprobe=3)
    alone = [ivf.search(q[r], 10, nprobe=3) for r in (0, 64, 150, 199)]
    monkeypatch.setattr(search, "IVF_SCRATCH_CAP", search.ivf_scratch_bytes(50, 3, ivf.nlist, len(ivf), 320, 10))
    assert search.ivf_query_batch(3, ivf.nlist, len(ivf), 320, 10) < 100
    split = ivf.search(q, 10, nprobe=3)
    assert torch.equal(whole[0], split[0]) and torch.equal(whole[1], split[1])
    for r, (s, i) in zip((0, 64, 150, 199), alone):
        assert torch.equal(s[0], whole[0][r]) and torch.equal(i[0], whole[1][r])


# ---- k-means ------------------------------------------------------------------------------------------------------------
def test_means_equal_the_exact_reference():
    from esm_b200 import search
    g = torch.Generator().manual_seed(9)
    for metric, scale in (("cosine", 1.0), ("l2", 3e4)):
        x = search.prepare_rows((torch.randn(5000, 200, generator=g) * scale).clamp(-65504, 65504), metric).to(DEV)
        a = torch.randint(-1, 37, (5000,), generator=g).to(DEV)  # -1: left out
        sums, means, counts = search.kmeans_means(x, a, 36)
        rs, rm, rc = ivf_refs.exact_means(x, a, 36)
        assert torch.equal(sums.cpu(), rs) and torch.equal(counts.cpu(), rc) and torch.equal(means.cpu(), rm)


def test_means_in_slices_equal_the_kernel(monkeypatch):
    from esm_b200 import search
    g = torch.Generator().manual_seed(16)
    x = search.prepare_rows((torch.randn(5000, 128, generator=g) * 3e4).clamp(-65504, 65504), "l2").to(DEV)
    a = torch.randint(-1, 20, (5000,), generator=g).to(DEV)
    _, want_means, want_counts = search.kmeans_means(x, a, 19)
    monkeypatch.setattr(search, "MEAN_ROWS", 1024)  # five slices, the last one short
    means, counts = search.exact_means(x, a, 19)
    assert torch.equal(means, want_means) and torch.equal(counts, want_counts)
    assert torch.equal(means.cpu(), ivf_refs.exact_means(x, a, 19)[1])


def _restated_training(x_rows, dim, metric, nlist, iters):
    """train_kmeans with the CPU exact-mean reference in place of the kernel; returns the centroids and how many
    clusters were refilled over the iterations."""
    from esm_b200 import search
    x_sqnorm = search.squared_norms(x_rows) if metric == "l2" else None
    cent, refilled = x_rows[:nlist].clone(), 0
    for _ in range(iters):
        s, a = search._assign(x_rows, cent, metric)
        got = search.kmeans_means(x_rows, a, nlist)
        want = ivf_refs.exact_means(x_rows, a, nlist)
        assert all(torch.equal(u.cpu(), v) for u, v in zip(got, want))
        means, counts = want[1].to(DEV), want[2].to(DEV)
        empty = counts == 0
        if metric == "cosine":
            empty |= (means != 0).sum(1) == 0
        refilled += int(empty.sum())
        new = torch.empty_like(cent)
        keep = (~empty).nonzero().flatten()
        new[keep] = search.prepare_rows(means[keep][:, :dim], metric)
        cent = search.fill_empty(new, empty, x_rows, s, x_sqnorm, metric)
    return cent, refilled


@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_training_matches_its_restatement_and_refills_empty_clusters(metric):
    from esm_b200 import search
    N, E, nlist, train = 4000, 100, 16, 2000
    x = torch.randn(N, E, generator=torch.Generator().manual_seed(10))
    sample = search.training_sample(N, train, 0)
    x[sample[1]] = x[sample[0]]  # two equal initial centroids: the second is empty after the first assignment
    x[sample[2]] = x[sample[0]]
    rows = search.prepare_rows(x, metric).to(DEV)
    want, refilled = _restated_training(rows[sample.to(DEV)], E, metric, nlist, 4)
    assert refilled >= 2
    got = search.train_kmeans(rows, E, metric, nlist, train, 4, 0)
    assert torch.equal(got, want)


def test_builds_are_deterministic():
    from esm_b200 import search
    x = torch.randn(6000, 128, generator=torch.Generator().manual_seed(11))
    a = search.IVFIndex(x, nlist=24, iters=5, seed=3)
    b = search.IVFIndex(x.to(DEV), nlist=24, iters=5, seed=3)
    for name in ("centroids", "ids", "offsets", "rows"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    assert int(a.offsets[-1]) == 6000 and torch.equal(torch.sort(a.ids).values.cpu(), torch.arange(6000))
    # each list holds its rows in ascending original index
    for l in range(24):
        seg = a.ids[a.offsets[l]:a.offsets[l + 1]]
        assert bool((seg[1:] > seg[:-1]).all())
    c = search.IVFIndex(x, nlist=24, iters=5, seed=4)
    assert not torch.equal(a.centroids, c.centroids)


def _mixture(n, E, centers, g, spread=0.05):
    c = torch.nn.functional.normalize(torch.randn(centers, E, generator=g), dim=1)
    lab = torch.randint(0, centers, (n,), generator=g)
    return c[lab] + spread * torch.randn(n, E, generator=g) / E ** 0.5


def test_recall_on_a_separated_mixture():
    from esm_b200 import search
    g = torch.Generator().manual_seed(12)
    x = _mixture(20000, 256, 64, g)
    q = _mixture(500, 256, 64, torch.Generator().manual_seed(12))  # the same centres
    exact = search.EmbeddingIndex(x).to(DEV)
    ivf = search.IVFIndex.from_index(exact, nlist=64, iters=10)
    _, want = exact.search(q, 10)
    _, got = ivf.search(q, 10, nprobe=4)
    recall = sum(len(set(a) & set(b)) for a, b in zip(want.tolist(), got.tolist())) / want.numel()
    assert recall >= 0.95, recall


# ---- CLI ----------------------------------------------------------------------------------------------------------------
def test_cli_ivf_with_every_list_writes_the_exact_hits(tmp_path):
    from esm_b200 import search_cli
    g = torch.Generator().manual_seed(13)
    for split in ("db", "queries"):
        for i in range(150 if split == "db" else 20):
            v = torch.randn(320, generator=g)
            (tmp_path / split).mkdir(exist_ok=True)
            torch.save({"label": f"{split}{i:03d}", "mean_representations": {33: v}}, tmp_path / split / f"{i}.pt")
    p = search_cli.create_parser()
    search_cli.run(p.parse_args(["build", str(tmp_path / "db"), "--layer", "33", "--out", str(tmp_path / "db.pt")]))
    search_cli.run(p.parse_args(["build", str(tmp_path / "db"), "--layer", "33", "--out", str(tmp_path / "ivf.pt"),
                                 "--nlist", "6", "--iters", "4"]))
    for src in (["--queries", str(tmp_path / "queries")], ["--all"]):
        search_cli.run(p.parse_args(["query", str(tmp_path / "db.pt"), *src, "--k", "7", "--out",
                                     str(tmp_path / "a.tsv")]))
        search_cli.run(p.parse_args(["query", str(tmp_path / "ivf.pt"), *src, "--k", "7", "--nprobe", "6", "--out",
                                     str(tmp_path / "b.tsv")]))
        assert (tmp_path / "a.tsv").read_text() == (tmp_path / "b.tsv").read_text()


# ---- refusals with real buffers -------------------------------------------------------------------------------------------
def test_refusals_with_real_buffers():
    from esm_b200 import _lib, search
    import test_ivf_host as host
    lib = _lib.load()
    buf = torch.zeros(1 << 24, dtype=torch.uint8, device=DEV)
    base = buf.data_ptr()
    for over, msg in host.IVF_REFUSALS:
        kw = dict(host.IVF_ARGS)
        for key, v in list(kw.items()):
            if v == host._FAKE:
                kw[key] = base
        for key, v in over.items():
            kw[key] = v if not isinstance(v, int) or v < host._FAKE or key in ("scratch_bytes", "Q", "N", "nlist",
                                                                               "nprobe", "k", "D", "q_ld", "b_ld") \
                else base + (v - host._FAKE)
        before = lib.esmb200_launch_count()
        rc = lib.esmb200_ivf_search(*kw.values(), None)
        assert rc == -1 and msg in lib.esmb200_last_error().decode(), (over, lib.esmb200_last_error())
        assert lib.esmb200_launch_count() == before
    for over, msg in host.MEANS_REFUSALS:
        kw = {key: (base if v == host._FAKE else v) for key, v in host.MEANS_ARGS.items()}
        for key, v in over.items():
            kw[key] = base + (v - host._FAKE) if isinstance(v, int) and v >= host._FAKE and key in (
                "rows", "assign") else v
        before = lib.esmb200_launch_count()
        rc = lib.esmb200_kmeans_means(*kw.values(), None)
        assert rc == -1 and msg in lib.esmb200_last_error().decode(), (over, lib.esmb200_last_error())
        assert lib.esmb200_launch_count() == before
