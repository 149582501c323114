"""GPU: embedding alignment (esm_b200.align, esmb200_align_similarity / esmb200_align).

  1. S and the z-scored S' against float64 on the kernel's own fp16 rows: S within the fp32 accumulation bound of its
     D fp16 products (ref.sim_bound); S' within that bound carried through the z-score (divided by the row and column
     standard deviations, x4 for the statistics' own error) plus 1e-5 (1 + |S'|) for the fp32 division and sum;
  2. the dynamic programme bit for bit against the float32 numpy restatement run on the GPU's own S': score bits, both
     spans and the op string, local and global;
  3. caller-chosen S' with ties (integer-valued matrices, o == e, zero penalties, constant matrices);
  4. row blocks past the warp (La = 1 ... 4,100, odd and prime, La >> Lb and La << Lb);
  5. mixed-length batches: a pair alone, inside a batch and under several max_cells gives the same result, and
     repeated runs are identical;
  6. every C-ABI refusal with real buffers, launching nothing;
  7. align_cli end to end on extract_cli output of a random-weight small ESM-2, its a3m read back by variants.read_msa
     and fed to MSATransformer.predict_contacts.
"""
import ctypes
import os
import struct
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # align_refs

import align_refs as ref  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _emb(lengths, E, seed):
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(max(lengths) + 8, E, generator=g)
    # related proteins: shifted, noisy windows of one base, so the alignments have structure to find
    out = []
    for k, L in enumerate(lengths):
        s = int(torch.randint(0, 8, (1,), generator=g))
        out.append(base[s:s + L] + 0.7 * torch.randn(L, E, generator=g))
    return out


def _bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


def _check_against_oracle(res, sims, mode, o, e):
    for p, (a, s) in enumerate(zip(res, sims)):
        want = ref.align(s.cpu().numpy(), mode, o, e)
        got = (a.score, a.query_span, a.target_span, a.ops)
        assert _bits(a.score) == _bits(float(want[0])) and got[1:] == tuple(want[1:]), (p, got, want)


# ---- 1. similarity -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("E", [100, 320, 1280])
def test_similarity_against_float64(E):
    from esm_b200 import align, search
    qs, ts = _emb([1, 37, 64, 65, 300], E, 1), _emb([5, 64, 129, 1, 250], E, 2)
    for zscore in (False, True):
        _, sims = align.align_pairs(qs, ts, zscore=zscore, return_similarity=True)
        for q, t, s in zip(qs, ts, sims):
            q16 = search.prepare_rows(q.to(DEV), "cosine").cpu()  # the rows the kernel read
            t16 = search.prepare_rows(t.to(DEV), "cosine").cpu()
            s64, bound = ref.sim_f64(q16, t16), ref.sim_bound(q16, t16)
            got = s.double().cpu()
            assert got.shape == s64.shape
            if not zscore:
                assert bool(((got - s64).abs() <= bound).all()), float(((got - s64).abs() / bound).max())
                continue
            want = ref.zscore_f64(s64)
            sr = s64.std(1, unbiased=False, keepdim=True)
            sc = s64.std(0, unbiased=False, keepdim=True)
            b = bound.max()
            tol = 4 * 0.5 * (torch.where(sr > 0, b / sr.clamp_min(1e-300), 0 * sr) +
                             torch.where(sc > 0, b / sc.clamp_min(1e-300), 0 * sc)) + 1e-5 * (1 + want.abs())
            assert bool(((got - want).abs() <= tol).all()), float(((got - want).abs() / tol).max())


# ---- 2. the programme on the GPU's own S' -----------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["local", "global"])
@pytest.mark.parametrize("zscore", [True, False])
def test_dp_bit_for_bit_on_the_gpu_similarity(mode, zscore):
    from esm_b200 import align
    qs, ts = _emb([1, 2, 31, 32, 33, 97, 250, 500], 320, 3), _emb([300, 33, 1, 64, 7, 101, 249, 480], 320, 4)
    o, e = (1.0, 0.1) if zscore else (0.05, 0.01)
    res, sims = align.align_pairs(qs, ts, mode, o, e, zscore=zscore, return_similarity=True)
    _check_against_oracle(res, sims, mode, o, e)
    for a, s in zip(res, sims):
        if a.ops:
            assert abs(ref.score_of(s.cpu().numpy(), a.ops, a.query_span[0], a.target_span[0], o, e) - a.score) <= \
                1e-3 * (1 + abs(a.score))


# ---- 3. caller-chosen S' with ties -------------------------------------------------------------------------------
def _tie_matrices():
    g = torch.Generator().manual_seed(5)
    mats = [torch.randint(-2, 3, (La, Lb), generator=g).float() for La, Lb in
            [(1, 1), (1, 9), (9, 1), (13, 17), (40, 33), (64, 65), (100, 3), (3, 100)]]
    mats += [torch.zeros(20, 30), torch.ones(20, 30), -torch.ones(7, 5), torch.eye(33), torch.full((1, 1), -1.0)]
    return mats


@pytest.mark.parametrize("mode", ["local", "global"])
@pytest.mark.parametrize("o,e", [(1.0, 1.0), (0.0, 0.0), (2.0, 0.5), (0.5, 0.0)])
def test_caller_chosen_similarity_with_ties(mode, o, e):
    from esm_b200 import align
    mats = _tie_matrices()
    _check_against_oracle(align.align_matrices(mats, mode, o, e), mats, mode, o, e)


# ---- 4. row blocks past the warp ------------------------------------------------------------------------------------
@pytest.mark.parametrize("La,Lb", [(4100, 5), (5, 4100), (4100, 1), (1, 4100), (1021, 997), (2053, 61),
                                   (32, 4099), (97, 33)])
def test_long_and_lopsided_pairs(La, Lb):
    from esm_b200 import align
    g = torch.Generator().manual_seed(La * 7 + Lb)
    mats = [torch.randn(La, Lb, generator=g), torch.randint(-3, 4, (La, Lb), generator=g).float()]
    for mode in ("local", "global"):
        _check_against_oracle(align.align_matrices(mats, mode, 1.0, 0.25), mats, mode, 1.0, 0.25)


# ---- 5. independence of batching, chunking and repetition ------------------------------------------------------------
def test_results_depend_only_on_the_pair():
    from esm_b200 import align
    lq, lt = [57, 1, 300, 129, 33, 800, 2, 64], [64, 211, 5, 129, 901, 77, 1, 63]
    qs, ts = _emb(lq, 480, 6), _emb(lt, 480, 7)
    for mode in ("local", "global"):
        full, sims = align.align_pairs(qs, ts, mode, return_similarity=True)
        alone = [align.align_pairs([q], [t], mode)[0] for q, t in zip(qs, ts)]
        assert full == alone
        cells = max(a * b for a, b in zip(lq, lt))
        for mc in (cells, cells + 1, 2 * cells, 10 ** 7):
            res, s2 = align.align_pairs(qs, ts, mode, max_cells=mc, return_similarity=True)
            assert res == full and all(torch.equal(x, y) for x, y in zip(sims, s2))
        rev = align.align_pairs(qs[::-1], ts[::-1], mode)
        assert rev[::-1] == full
        for _ in range(3):
            assert align.align_pairs(qs, ts, mode) == full
        with pytest.raises(ValueError, match="max_cells"):
            align.align_pairs(qs, ts, mode, max_cells=cells - 1)


# ---- 6. refusals with real buffers ------------------------------------------------------------------------------
def test_c_abi_refusals_launch_nothing():
    from esm_b200 import _lib
    from esm_b200.model import _ptr
    lib = _lib.load()
    P, La, Lb = 2, 5, 7
    off_q = torch.tensor([0, La, 2 * La], dtype=torch.int64, device=DEV)
    off_t = torch.tensor([0, Lb, 2 * Lb], dtype=torch.int64, device=DEV)
    off_s = torch.tensor([0, La * Lb, 2 * La * Lb], dtype=torch.int64, device=DEV)
    nq, nt, nc = 2 * La, 2 * Lb, 2 * La * Lb
    need = lib.esmb200_align_scratch_bytes(P, nq, nt, nc)
    scratch = torch.empty(need, dtype=torch.uint8, device=DEV)
    s = torch.zeros(nc, device=DEV)
    q16 = torch.zeros(nq, 64, dtype=torch.float16, device=DEV)
    t16 = torch.zeros(nt, 64, dtype=torch.float16, device=DEV)
    scores, spans = torch.empty(P, device=DEV), torch.empty(P, 4, dtype=torch.int32, device=DEV)
    ops, n_ops = torch.empty(nq + nt, dtype=torch.uint8, device=DEV), torch.empty(P, dtype=torch.int32, device=DEV)
    base = dict(s=_ptr(s), q=_ptr(off_q), t=_ptr(off_t), so=_ptr(off_s), P=P, nq=nq, nt=nt, nc=nc, mode=0, o=1.0,
                e=0.1, scratch=_ptr(scratch), sb=need, scores=_ptr(scores), spans=_ptr(spans), ops=_ptr(ops),
                n_ops=_ptr(n_ops), stream=None)
    bad = [({"mode": 2}, "mode"), ({"o": float("nan")}, "penalties"), ({"e": -1.0}, "penalties"),
           ({"o": float("inf")}, "penalties"), ({"P": -1}, "P >= 0"), ({"nq": 1}, "n_q"), ({"nc": 1}, "n_q"),
           ({"sb": need - 1}, "more cells than the scratch"), ({"s": None}, "null"), ({"ops": None}, "null"),
           ({"scratch": ctypes.c_void_p(scratch.data_ptr() + 8)}, "256-byte")]
    before = lib.esmb200_launch_count()
    for over, msg in bad:
        rc = lib.esmb200_align(*dict(base, **over).values())
        assert rc == -1 and msg in lib.esmb200_last_error().decode(), (over, lib.esmb200_last_error())
    sim = dict(q=_ptr(q16), t=_ptr(t16), D=64, qo=_ptr(off_q), to=_ptr(off_t), so=_ptr(off_s), P=P, nq=nq, nt=nt,
               nc=nc, z=1, out=_ptr(s), scratch=_ptr(scratch), sb=need, stream=None)
    for over, msg in [({"D": 100}, "D % 64"), ({"z": 2}, "zscore"), ({"sb": 0}, "more cells"), ({"out": None}, "null"),
                      ({"q": ctypes.c_void_p(q16.data_ptr() + 2)}, "16-byte")]:
        rc = lib.esmb200_align_similarity(*dict(sim, **over).values())
        assert rc == -1 and msg in lib.esmb200_last_error().decode(), (over, lib.esmb200_last_error())
    assert lib.esmb200_launch_count() == before
    assert lib.esmb200_align(*dict(base, P=0, nq=0, nt=0, nc=0).values()) == 0 and lib.esmb200_launch_count() == before
    assert lib.esmb200_align(*base.values()) == 0
    torch.cuda.synchronize()
    assert lib.esmb200_launch_count() == before + 2


# ---- 7. the command line ------------------------------------------------------------------------------------------
def test_cli_end_to_end_into_the_msa_transformer(tmp_path):
    from esm_b200 import align, align_cli, extract_cli, pretrained, search_cli, variants
    from oracle.weights import make_state_dict
    L, E, H = 2, 128, 2
    sd = make_state_dict(L, E, H, seed=3)  # a random-weight small ESM-2 checkpoint
    ckpt = tmp_path / "esm2_small.pt"
    torch.save({"cfg": {"model": {"encoder_layers": L, "encoder_embed_dim": E, "encoder_attention_heads": H,
                                  "token_dropout": True}},
                "model": {("encoder.sentence_encoder." + k): v for k, v in sd.items()}}, ckpt)
    rng = np.random.default_rng(0)
    aa = np.array(list("ACDEFGHIKLMNPQRSTVWY"))
    core = "".join(rng.choice(aa, 60))
    seqs = {"q/a": core, "q/b": "".join(rng.choice(aa, 45))}
    for k in range(6):
        s = list(core[rng.integers(0, 10):])
        for _ in range(5):
            s[rng.integers(0, len(s))] = rng.choice(aa)
        seqs[f"t{k}"] = "".join(rng.choice(aa, rng.integers(0, 6))) + "".join(s)
    fasta = tmp_path / "all.fasta"
    fasta.write_text("".join(f">{k}\n{v}\n" for k, v in seqs.items()))
    out = tmp_path / "emb"
    p = extract_cli.create_parser()
    assert extract_cli.run(p.parse_args([str(ckpt), str(fasta), str(out), "--include", "mean", "per_tok",
                                         "--repr_layers", str(L)])) == len(seqs)
    sp = search_cli.create_parser()
    search_cli.run(sp.parse_args(["build", str(out), "--layer", str(L), "--out", str(tmp_path / "db.pt")]))
    search_cli.run(sp.parse_args(["query", str(tmp_path / "db.pt"), "--all", "--k", "4",
                                  "--out", str(tmp_path / "hits.tsv")]))
    ap = align_cli.create_parser()
    n = align_cli.run(ap.parse_args([str(tmp_path / "hits.tsv"), "--queries", str(out), "--targets", str(out),
                                     "--layer", str(L), "--out", str(tmp_path / "aln.tsv"), "--fasta", str(fasta),
                                     "--a3m", str(tmp_path / "a3m")]))
    assert n == 4 * len(seqs)
    hits = align_cli.read_hits(tmp_path / "hits.tsv")
    lines = (tmp_path / "aln.tsv").read_text().splitlines()
    assert len(lines) == n + 1 and lines[0].split("\t")[:5] == ["query", "rank", "target", "search_score", "score"]
    emb = {k: torch.load(out / f"{k}.pt", weights_only=True)["representations"][L] for k in seqs}
    want = align.align_pairs([emb[h[0]] for h in hits], [emb[h[2]] for h in hits])
    for line, h, a in zip(lines[1:], hits, want):
        f = line.split("\t")
        assert f[:3] == [h[0], str(h[1]), h[2]] and f[3] == h[3]
        assert f[4:] == [f"{a.score:.6g}", str(a.query_span[0]), str(a.query_span[1]), str(a.target_span[0]),
                         str(a.target_span[1]), a.cigar()]
    model, alphabet = pretrained.esm_msa1b_t12_100M_UR50S(allow_random_init=True)
    model = model.eval().cuda()
    for q in seqs:
        rows = variants.read_msa(tmp_path / "a3m" / f"{q}.a3m", None)
        assert len(rows) == 5 and rows[0] == (q, seqs[q]) and all(len(r[1]) == len(seqs[q]) for r in rows)
        assert [r[0] for r in rows[1:]] == [h[2] for h in hits if h[0] == q]
        _, _, tokens = alphabet.get_batch_converter()(rows)
        c = model.predict_contacts(tokens.cuda())
        assert c.shape == (1, len(seqs[q]), len(seqs[q])) and bool(torch.isfinite(c).all())
