"""GPU: greedy row selection for the MSA Transformer (esm_b200.msa_select, esmb200_msa_greedy_select).

  1. the rows of every case of tests/golden/msa_select.json (the reference notebook's greedy_select), both modes;
  2. the selection order against the numpy restatement (tests/msa_select_refs.py), bit for bit, up to 50,000 rows,
     columns that are not a multiple of 16 (padded on the device), one column, a row wider than 48 KiB and picks past
     128, 256 and 512; past the step kernel's 256 partials and the init kernel's grid (N = 70,000 and 300,000) with
     poisoned scratch, scratch reused by a second call, a count of 65,535 and k = N, through the C ABI;
  3. the tensor API under torch.cuda.set_sync_debug_mode("error");
  4. every argument refusal of the C ABI, before any launch;
  5. predict_cli and sample_msa_cli with --msa-select against the same commands on an a3m file that holds exactly the
     picked rows.
"""
import ctypes
import functools
import json
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # msa_select_refs, variant_fixtures

import msa_select_refs as ref  # noqa: E402

pytestmark = pytest.mark.gpu


def _random_rows(N, C, symbols, seed):
    g = np.random.default_rng(seed)
    alphabet = np.frombuffer(b"ACDEFGHIKLMNPQRSTVWY-", dtype=np.uint8)[:symbols]
    return alphabet[g.integers(0, symbols, (N, C))]


# ---- 1. the notebook's rows ----------------------------------------------------------------------------------------
def test_the_rows_equal_the_notebook_on_every_fixture_case():
    from esm_b200 import msa_select
    cases = ref.fixture_cases()
    for msa, k, mode, selected in cases:
        assert msa_select.greedy_select(msa, k, mode) == [msa[i] for i in selected], (len(msa), k, mode)
        if len(msa) > k > 1:
            idx = msa_select.greedy_select_indices(torch.from_numpy(ref.as_rows(msa)).cuda(), k, mode)
            assert idx.is_cuda and idx.dtype == torch.int64 and idx.tolist() == selected
    print(f"PARITY msa_select: {len(cases)} fixture cases pick the notebook's rows in both modes", flush=True)


# ---- 2. the selection order ----------------------------------------------------------------------------------------
ORDER_CASES = [  # N, C, k, symbols
    (50000, 37, 40, 3),
    (20000, 100, 140, 21),
    (3000, 1, 300, 2),
    (4099, 65, 260, 2),
    (1500, 7, 600, 3),
    (300, 50000, 12, 2),  # the picked row needs more than 48 KiB of shared memory
]


@pytest.mark.parametrize("N,C,k,symbols", ORDER_CASES)
@pytest.mark.parametrize("mode", ["max", "min"])
def test_the_selection_order_matches_the_restatement(N, C, k, symbols, mode):
    from esm_b200 import msa_select
    rows = _random_rows(N, C, symbols, seed=N + C + k)
    want = ref.greedy_order(rows, k, mode)
    got = msa_select._order(torch.from_numpy(rows).cuda(), k, mode).tolist()
    assert got == want
    print(f"PARITY msa_select order N={N} C={C} k={k} {mode}: equal to the restatement", flush=True)


# ---- 2b. past the grid caps, through the C ABI with poisoned scratch ------------------------------------------------
def _select_abi(rows, C, k, mode, scratch=None):
    """esmb200_msa_greedy_select on rows uint8 [N, ld] (contiguous on the GPU, ld a multiple of 16). The scratch, when
    not given, is filled with 0xFF bytes first: every row then reads as picked and every table entry as NaN until the
    init kernel rewrites it. Returns (the picks, the scratch)."""
    from esm_b200 import _lib
    lib = _lib.load()
    N, ld = rows.shape
    n = lib.esmb200_msa_select_scratch_bytes(N, C, k)
    if scratch is None:
        scratch = torch.full((n,), 0xFF, dtype=torch.uint8, device="cuda")
    assert scratch.numel() >= n
    sel = torch.full((k,), -1, dtype=torch.int64, device="cuda")
    code = _lib.SELECT_MAX if mode == "max" else _lib.SELECT_MIN
    _lib.check(lib.esmb200_msa_greedy_select(rows.data_ptr(), ld, N, C, k, code, sel.data_ptr(), scratch.data_ptr(),
                                             scratch.numel(), torch.cuda.current_stream().cuda_stream))
    return sel.tolist(), scratch


FAR = (65536, 262144)  # the step kernel's 256 partials per last-block pass, and the init kernel's 1024 x 256 grid
SCALE_C, SCALE_K = 48, 48


@functools.lru_cache(maxsize=None)
def _scale_case(N, mode):
    """Random rows over four letters, and 8 planted rows in each of [65536, 262144) and [262144, N) that win the first
    picks: in max mode rows over sixteen other letters (they differ from every other row in every column), in min
    mode near-copies of the query (1 to 4 columns changed). Random rows tie often and ties go to the smallest index,
    so without them the picks could all come from the first blocks. Returns (rows, the restatement's picks)."""
    rows = _random_rows(N, SCALE_C, 4, seed=N + (mode == "min"))
    g = np.random.default_rng(N + 7)
    planted = np.concatenate([g.choice(np.arange(lo, min(hi, N)), 8, replace=False)
                              for lo, hi in zip(FAR, FAR[1:] + (N,)) if lo < N])
    other = np.frombuffer(b"FGHIKLMNPQRSTVWY", dtype=np.uint8)
    for m, r in enumerate(planted):
        if mode == "max":
            rows[r] = other[g.integers(0, 16, SCALE_C)]
        else:
            rows[r] = rows[0]
            cols = g.choice(SCALE_C, 1 + m % 4, replace=False)
            rows[r, cols] = np.where(rows[0, cols] == ord("A"), ord("C"), ord("A"))
    return rows, ref.greedy_order(rows, SCALE_K, mode)


def _far_picks(want, N):
    """The restatement's picks in [65536, 262144) and past 262144: each range that N reaches must hold some."""
    far = [sum(FAR[0] <= i < FAR[1] for i in want), sum(i >= FAR[1] for i in want)]
    assert far[0] > 0 and (N <= FAR[1] or far[1] > 0), want
    return far


@pytest.mark.parametrize("mode", ["max", "min"])
@pytest.mark.parametrize("N", [70000, 300000])
def test_the_selection_order_past_the_grid_caps(N, mode):
    """N = 70,000 has 274 blocks, so the last block's loop over the partials runs twice; N = 300,000 also needs the
    init kernel's grid-stride loop (1172 blocks of rows against its 1024)."""
    rows, want = _scale_case(N, mode)
    far = _far_picks(want, N)
    got, _ = _select_abi(torch.from_numpy(rows).cuda(), SCALE_C, SCALE_K, mode)
    print(f"PARITY msa_select order N={N} C={SCALE_C} k={SCALE_K} {mode}, poisoned scratch: "
          f"{'equal to' if got == want else 'DIFFERENT from'} the restatement; picks past 65,536 / 262,144: "
          f"{far[0]} / {far[1]}", flush=True)
    assert got == want


def test_scratch_reused_for_a_smaller_alignment_and_the_other_mode():
    """The init kernel rewrites picked, the distance table and the ticket: a second call on the first call's scratch,
    with fewer rows (so every array sits at another offset) and the other mode, picks the restatement's rows too."""
    (big, want_big), (small, want_small) = _scale_case(300000, "max"), _scale_case(70000, "min")
    got_big, scratch = _select_abi(torch.from_numpy(big).cuda(), SCALE_C, SCALE_K, "max")
    got_small, _ = _select_abi(torch.from_numpy(small).cuda(), SCALE_C, SCALE_K, "min", scratch=scratch)
    print(f"PARITY msa_select scratch reuse: N=300000 max then N=70000 min on one scratch, "
          f"{'both equal' if (got_big, got_small) == (want_big, want_small) else 'NOT equal'} to the restatement",
          flush=True)
    assert got_big == want_big and got_small == want_small


def test_the_count_at_its_maximum():
    """C = 65,535 and a row that differs from the query in every column: its uint16 count is 65,535, its distance
    exactly 1.0, so max mode picks it first."""
    N, C, k, far = 200, 65535, 12, 137
    rows = _random_rows(N, C, 4, seed=C)
    rows[far] = ord("W")
    ld = C + 1
    dev = torch.zeros((N, ld), dtype=torch.uint8, device="cuda")
    dev[:, :C] = torch.from_numpy(rows).cuda()
    for mode in ("max", "min"):
        got, scratch = _select_abi(dev, C, k, mode)
        counts = scratch[:2 * N].view(torch.int16).cpu().numpy().view(np.uint16)  # counts[0, :]: against the query
        assert counts[far] == 65535 and np.array_equal(counts, (rows != rows[0]).sum(1))
        want = ref.greedy_order(rows, k, mode)
        assert got == want
        if mode == "max":
            assert want[1] == far
    print(f"PARITY msa_select C={C} N={N} k={k}: count {int(counts[far])} (d = 1.0) picked second in max mode; both "
          f"modes equal to the restatement", flush=True)


@pytest.mark.parametrize("mode", ["max", "min"])
def test_k_equal_to_n_runs_to_a_single_candidate(mode):
    """The C ABI at k = N: the last step has one unpicked row left. The Python API returns every row without a launch
    there, so this compares with the restatement's loop run to k = N."""
    N, C = 600, 32
    rows = _random_rows(N, C, 3, seed=N + C)
    got, _ = _select_abi(torch.from_numpy(rows).cuda(), C, N, mode)
    want = ref.greedy_order(rows, N, mode, shortcut=False)
    print(f"PARITY msa_select k=N={N} C={C} {mode}: {'equal to' if got == want else 'DIFFERENT from'} the "
          f"restatement's loop without the N <= k shortcut", flush=True)
    assert got == want and sorted(got) == list(range(N))


# ---- 3. host synchronisation ---------------------------------------------------------------------------------------
def test_the_tensor_api_never_synchronises():
    from esm_b200 import msa_select
    rows = _random_rows(10000, 100, 21, seed=9)
    dev = torch.from_numpy(rows).cuda()
    msa_select.greedy_select_indices(dev, 8, "max")  # loads the library and warms the allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        a = msa_select.greedy_select_indices(dev, 200, "max")
        b = msa_select.greedy_select_indices(dev, 200, "min")
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert a.tolist() == sorted(ref.greedy_order(rows, 200, "max"))
    assert b.tolist() == sorted(ref.greedy_order(rows, 200, "min"))


# ---- 4. refusals ---------------------------------------------------------------------------------------------------
def test_every_refusal_comes_before_any_launch():
    from esm_b200 import _lib
    lib = _lib.load()
    N, C, k = 100, 20, 10
    rows = torch.zeros((N, 32), dtype=torch.uint8, device="cuda")
    sel = torch.empty(k, dtype=torch.int64, device="cuda")
    nbytes = lib.esmb200_msa_select_scratch_bytes(N, C, k)
    scratch = torch.empty(nbytes + 512, dtype=torch.uint8, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)  # noqa: E731
    good = dict(rows=p(rows), ld=32, N=N, C=C, k=k, mode=_lib.SELECT_MAX, sel=p(sel), scratch=p(scratch),
                nbytes=nbytes)
    bad = [dict(C=0), dict(C=65536, ld=65536), dict(k=N + 1), dict(k=-1), dict(N=-1), dict(mode=2), dict(mode=-1),
           dict(nbytes=nbytes - 1), dict(ld=16), dict(ld=40), dict(rows=p(rows, 8)), dict(scratch=p(scratch, 128)),
           dict(rows=None), dict(sel=None), dict(scratch=None)]
    before = lib.esmb200_launch_count()
    for change in bad:
        a = dict(good, **change)
        rc = lib.esmb200_msa_greedy_select(a["rows"], a["ld"], a["N"], a["C"], a["k"], a["mode"], a["sel"],
                                           a["scratch"], a["nbytes"], st)
        assert rc == -1, change  # ESMB200_EINVAL
    assert lib.esmb200_launch_count() == before
    a = good
    assert lib.esmb200_msa_greedy_select(a["rows"], a["ld"], a["N"], a["C"], 0, a["mode"], None, None, 0, st) == 0
    assert lib.esmb200_launch_count() == before  # k == 0 launches nothing
    _lib.check(lib.esmb200_msa_greedy_select(a["rows"], a["ld"], a["N"], a["C"], a["k"], a["mode"], a["sel"],
                                             a["scratch"], a["nbytes"], st))
    assert lib.esmb200_launch_count() == before + k  # the init kernel and one per step
    assert sel.tolist() == list(range(k))  # all rows equal: every tie goes to the smallest index


# ---- 5. the command lines ------------------------------------------------------------------------------------------
def _deep_a3m(a3m, n_extra, seed, tmp_path):
    """The variant fixture's alignment and n_extra seeded variants of its rows, without insertions."""
    from esm_b200 import variants
    (tmp_path / "in.a3m").write_text(a3m)
    msa = variants.read_msa(tmp_path / "in.a3m", None)
    g = np.random.default_rng(seed)
    letters = list("ACDEFGHIKLMNPQRSTVWY-")
    for i in range(n_extra):
        row = list(msa[g.integers(0, len(msa))][1])
        for j in g.choice(len(row), len(row) // 3, replace=False):
            row[j] = letters[g.integers(0, len(letters))]
        msa.append((f"variant{i}", "".join(row)))
    return msa


def _write_a3m(path, msa):
    path.write_text("".join(f">{d}\n{s}\n" for d, s in msa))


@pytest.fixture(scope="module")
def cli_inputs(golden_dir, tmp_path_factory):
    with open(os.path.join(golden_dir, "variants.json")) as f:
        fx = json.load(f)
    return fx, _deep_a3m(fx["a3m"], 30, 11, tmp_path_factory.mktemp("msa"))


@pytest.mark.parametrize("mode", ["max", "min"])
def test_predict_cli_scores_the_picked_rows(cli_inputs, tmp_path, mode):
    import variant_fixtures as vf
    from esm_b200 import msa_select, predict_cli
    fx, msa = cli_inputs
    _write_a3m(tmp_path / "full.a3m", msa)
    picked = msa_select.greedy_select(msa, 9, mode)
    assert picked != msa[:9]
    _write_a3m(tmp_path / "picked.a3m", picked)
    (tmp_path / "dms.csv").write_text(fx["dms_csv"])
    path = vf.write_checkpoint("msa_t2_tiny", vf.MODELS["msa_t2_tiny"], str(tmp_path))

    def run(a3m, out, extra):
        predict_cli.run(predict_cli.create_parser().parse_args(
            ["--model-location", path, "--sequence", fx["sequence"], "--dms-input", str(tmp_path / "dms.csv"),
             "--dms-output", str(out), "--offset-idx", str(fx["offset_idx"]), "--scoring-strategy", "masked-marginals",
             "--msa-path", str(a3m), "--msa-samples", "9"] + extra))
        return out.read_text()

    got = run(tmp_path / "full.a3m", tmp_path / "selected.csv", ["--msa-select", mode])
    want = run(tmp_path / "picked.a3m", tmp_path / "want.csv", [])
    assert got == want
    assert run(tmp_path / "full.a3m", tmp_path / "first.csv", []) != got
    print(f"PARITY predict_cli --msa-select {mode}: the CSV of the picked rows", flush=True)


def test_sample_msa_cli_samples_the_picked_rows(cli_inputs, tmp_path):
    import variant_fixtures as vf
    from esm_b200 import msa_select, sample_msa_cli
    _, msa = cli_inputs
    _write_a3m(tmp_path / "full.a3m", msa)
    picked = msa_select.greedy_select(msa, 9, "max")
    _write_a3m(tmp_path / "picked.a3m", picked)
    path = vf.write_checkpoint("msa_t2_tiny", vf.MODELS["msa_t2_tiny"], str(tmp_path))
    common = ["--append-rows", "2", "--chains", "2", "--sweeps", "1", "--block", "6", "--seed", "5"]
    p = sample_msa_cli.create_parser()
    sample_msa_cli.run(p.parse_args([path, "--msa", str(tmp_path / "full.a3m"), "--msa-samples", "9",
                                     "--msa-select", "max", "--out", str(tmp_path / "a")] + common))
    sample_msa_cli.run(p.parse_args([path, "--msa", str(tmp_path / "picked.a3m"), "--out", str(tmp_path / "b")] +
                                    common))
    for name in ["samples.tsv", "sample_0.a3m", "sample_1.a3m"]:
        assert (tmp_path / "a" / name).read_text() == (tmp_path / "b" / name).read_text(), name
    print("PARITY sample_msa_cli --msa-select max: the samples of the picked rows", flush=True)
