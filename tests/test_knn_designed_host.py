"""CPU: the designed exact-score databases of tests/test_gpu_knn_designed.py and the restatement of the top-k kernel's
queue protocol (search_refs.queue_protocol) they are checked with.

  1. the restatement's final lists equal the exact top k (float64 sort, search_refs.topk_exact) on random, tied and
     designed scores, across splits and a seeded running list;
  2. the keys decode back to their scores and indices, -0 to +0, key 0 to NaN and 2^32 - 1;
  3. each design reaches the queue counts, merges and skips it names, for every k the GPU file runs: a queue of
     exactly 64, 31 then a full chunk, 33, a row merged because another row overflowed, thresholds rising mid-tile,
     skipped tiles between busy ones, and a survivor in every epilogue register slot of both row halves.
"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import search_refs as ref  # noqa: E402

KS = [1, 31, 32, 33, 64, 127, 128]


def _via_protocol(s, mask, k, splits=1, seed=None):
    b = ref.biased_keys(s, mask).numpy()
    return torch.from_numpy(ref.queue_protocol(b, k, splits, seed))


def _exact(s, mask, k):
    """topk_exact, the float64 stable sort, in the form of decoded keys."""
    es, ei = ref.topk_exact(s, k, mask)
    return es.float() + 0.0, ei


@pytest.mark.parametrize("splits", [1, 2, 7])
@pytest.mark.parametrize("k", [1, 33, 128])
def test_the_protocol_reproduces_the_exact_top_k(k, splits):
    g = torch.Generator().manual_seed(k + splits)
    cases = [torch.randn(70, 1500, generator=g).float().double(),
             torch.randint(-2, 3, (70, 1500), generator=g).double()]  # ties everywhere
    hi, lo = ref.schedule_design()
    cases.append((hi + lo)[:, :1500])
    for s in cases:
        mask = ref.candidates_mask(s.shape[0], s.shape[1], 3, s.device)
        got_s, got_i = ref.decode(_via_protocol(s, mask, k, splits))
        es, ei = _exact(s, mask, k)
        assert torch.equal(got_i, ei) and torch.equal(got_s, es.float())
        assert torch.equal(got_i, ref.designed_topk(s, k, mask)[1])


def test_a_seeded_running_list_gives_the_top_k_of_both():
    g = torch.Generator().manual_seed(3)
    s = torch.randint(-50, 50, (64, 2000), generator=g).double()
    mask = torch.ones_like(s, dtype=torch.bool)
    b = ref.biased_keys(s, mask)
    for k in (1, 40, 128):
        seed = ref.top_keys(b[:, :700], k).numpy()  # the running list after rows [0, 700)
        got = torch.from_numpy(ref.queue_protocol(b[:, 700:].numpy(), k, 3, seed))
        assert torch.equal(got, ref.top_keys(b, k))


def test_keys_decode_to_scores_and_indices():
    s = torch.tensor([[0.0, -0.0, 1.5, -2.0, float("inf"), -float("inf"), ref.FLT_MAX, -ref.FLT_MAX, 2.0 ** -149,
                       -(2.0 ** -149), 2.0 ** -126 - 2.0 ** -149]], dtype=torch.float64)
    mask = torch.ones_like(s, dtype=torch.bool)
    mask[0, 3] = False
    row0 = (1 << 31) - 1 - s.shape[1]
    b = ref.biased_keys(s, mask, row0)
    sc, ix = ref.decode(b)
    keep = mask[0]
    assert torch.equal(sc[0, keep], (s[0, keep].float() + 0.0))
    assert torch.equal(ix[0, keep], torch.arange(s.shape[1])[keep] + row0)
    assert int(sc[0, 1].view(torch.int32)) == 0  # -0 ranks and decodes as +0
    assert int(sc[0, 3].view(torch.int32)) == -1 and int(ix[0, 3]) == (1 << 32) - 1  # key 0: the empty slot
    # the order of keys is (score descending, index ascending); -inf is above the empty slot
    order = torch.argsort(b[0], descending=True)
    assert order.tolist() == [4, 6, 2, 10, 8, 0, 1, 9, 7, 5, 3]
    assert torch.equal(ref.raw_keys(b)[0, 3], torch.tensor(0))
    with pytest.raises(AssertionError, match="not exact in fp32"):
        ref.biased_keys(torch.tensor([[0.1]], dtype=torch.float64), torch.ones(1, 1, dtype=torch.bool))


def test_materialize_gives_the_designed_scores():
    hi, lo = ref.schedule_design()
    for Q in (1, 65, 200):
        A, X, s = ref.materialize(hi, lo, 256, Q)
        assert torch.equal(A.double() @ X.double().T, s)
        # the two slots of every query lie in different 64-wide K blocks
        cols = [torch.nonzero(a).flatten().tolist() for a in A[:3]]
        assert all(len(c) == 2 and c[0] // 64 != c[1] // 64 for c in cols)
    A, X, s = ref.materialize(torch.randint(-2048, 2049, (64, 300)).double(), None, 64, 64)
    assert torch.equal(A.double() @ X.double().T, s)


# ---- the designs reach what they name ------------------------------------------------------------------------------
def _schedule_trace(k, Q=64):
    hi, lo = ref.schedule_design()
    _, _, s = ref.materialize(hi, lo, 256, Q)
    mask = torch.ones_like(s, dtype=torch.bool)
    trace = ref.Trace()
    got = ref.queue_protocol(ref.biased_keys(s, mask).numpy(), k, 1, trace=trace)
    assert torch.equal(torch.from_numpy(got), ref.top_keys(ref.biased_keys(s, mask), k))
    return trace


@pytest.mark.parametrize("k", KS)
def test_the_schedule_design_reaches_every_queue_edge(k):
    tr = _schedule_trace(k)
    block0 = [c for c in tr.chunks if c["block"] == 0]
    after = [c["before"] + c["pushed"] for c in block0]
    # a queue of exactly 64: 32 queued, then a full chunk (row 8); 31 then a full chunk (row 0)
    assert any(c["before"][8] == 32 and c["pushed"][8] == 32 for c in block0)
    assert any(c["before"][0] == 31 and c["pushed"][0] == 32 for c in block0)
    # 33: a merge that only row 2 forces, at 33 entries
    assert any(c["merge"] and a[2] == 33 and (np.delete(a, 2) <= 32).all() for c, a in zip(block0, after))
    # rows merged with a short queue because another row overflowed: row 1 with 1 entry, row 5 with 32
    for row, n in ((1, 1), (5, 32)):
        assert any(c["merge"] and a[row] == n for c, a in zip(block0, after)), row
    # the threshold rises inside a tile: a merge at chunk < 7, then a survivor later in the same tile
    rises = [(c["tile"], c["chunk"]) for c in block0 if c["merge"] and c["chunk"] < 7]
    assert any(c["tile"] == t and c["chunk"] > ch and c["pushed"].sum() > 0 for t, ch in rises for c in block0)
    # tiles 3 and 5 hold no survivor for block 0 and are skipped between busy tiles
    skipped = {t for b, _, t in tr.skipped if b == 0}
    busy = {t for b, _, t in tr.busy if b == 0}
    assert {3, 5} <= skipped and {2, 4, 6} <= busy
    # every (i, c, e) register slot of the epilogue, for rows of both halves (hr = 0, 1), holds a survivor
    assert tr.slots.all()
    # no queue ever holds more than 64 (queue_protocol asserts it) and the protocol merges at the end
    assert max(int(a.max()) for a in after) == 64


@pytest.mark.parametrize("k", KS)
def test_the_schedule_records_are_the_only_survivors_past_the_warm_up(k):
    """Past tile 0, a chunk pushes exactly the records placed in it: the counts the design plans are the counts the
    kernel's queues see."""
    tr = _schedule_trace(k)
    rec = ref.schedule_records()
    for c in tr.chunks:
        if c["block"] != 0 or c["tile"] == 0:
            continue
        g = ref.TILE // ref.CHUNK * c["tile"] + c["chunk"]
        want = np.array([len(rec[r].get(g, [])) for r in range(64)])
        assert (c["pushed"] == want).all(), (c["tile"], c["chunk"])


def test_the_tie_design_cuts_through_its_boundary_ties():
    hi, lo = ref.tie_design()
    s = hi + lo
    mask = torch.ones_like(s, dtype=torch.bool)
    for k in (1, 5, 11, len(ref.TIE_COLUMNS)):
        _, idx = ref.designed_topk(s, k, mask)
        assert (idx == torch.tensor(ref.TIE_COLUMNS[:k])).all()
    _, idx = ref.designed_topk(s, 60, mask)
    top = s.gather(1, idx)
    assert bool((top[:, 16:] == 1.5).all())  # past the boundary columns, ties at 1.5 to the smaller index
    for splits in (1, 3):
        assert torch.equal(_via_protocol(s, mask, 60, splits), ref.top_keys(ref.biased_keys(s, mask), 60))
