"""GPU: alignment sampling from the MSA Transformer (esm_b200.sampling.msa_gibbs, esmb200_sample_order,
esmb200_sample_rows).

  1. the order kernel against the numpy restatement, bit for bit, up to entry 2^20 - 1 and chain0 near 2^32;
  2. the token-set sampler against float64 for 1, 20, 21 and 32 tokens: draws away from near-ties, log q bit for bit
     against esmb200_log_softmax_rows, ties to the smaller a, an out-of-range entry, the block sums;
  3. a chi-square test of 200,000 draws over the 21-token set;
  4. msa_gibbs on the tiny MSA fixture in fp16 and fp32x3: fixed entries, drawable tokens, chunking, seeds, and every
     step replayed through the public forward and the float64 Gumbel restatement;
  5. one step's logits against the float64 oracle, and the draws wherever the Gumbel gap exceeds that error;
  6. no host synchronisation after the first step;
  7. the command line end to end.
Every gated comparison prints a PARITY line.
"""
import json
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # sampling_refs, variant_fixtures

import sampling_refs as sr  # noqa: E402

pytestmark = pytest.mark.gpu

AA = list(range(4, 24))  # jacobian.AMINO_ACIDS in the MSA alphabet
GAP = 30
NEAR_TIE = 1e-5


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _tempered(logits, tau):
    """logits / fp32(tau) by IEEE fp32 division, as the kernel divides."""
    return logits / torch.full_like(logits, tau)


def _rows(logits, token_set, tau, seed, step, chain0, per, entries, tokens, R, C, logp=None, stride=0):
    from esm_b200 import _lib
    n = logits.shape[0]
    ts = torch.tensor(token_set, dtype=torch.int32, device="cuda")
    logq = torch.full((n,), float("nan"), device="cuda")
    _lib.check(_lib.load().esmb200_sample_rows(
        logits.data_ptr(), logits.stride(0), n, ts.data_ptr(), len(token_set), tau, seed, step, chain0, per,
        entries.data_ptr(), tokens.data_ptr(), tokens[0].numel(), R, C, logq.data_ptr(),
        logp.data_ptr() if logp is not None else None, stride, _stream()))
    return logq


# ---- 1. the order kernel --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,chains,chain0", [(1, 1, 0), (37, 5, 2 ** 32 - 5), (4093, 9, 3)])
def test_sample_order_of_alignment_entries_matches_the_restatement(n, chains, chain0):
    from esm_b200 import _lib
    entries = np.random.default_rng(n).choice(1 << 20, n, replace=False)
    entries[0] = (1 << 20) - 1
    ent = torch.as_tensor(entries, device="cuda")
    keys = torch.empty((chains, n), dtype=torch.int64, device="cuda")
    for sweep, seed in [(0, 0), (9, 2 ** 64 - 1), (2 ** 32 - 1, 77)]:
        _lib.check(_lib.load().esmb200_sample_order(ent.data_ptr(), n, chains, chain0, sweep, seed, keys.data_ptr(),
                                                    _stream()))
        want = sr.order_keys(entries, chain0 + np.arange(chains), sweep, seed)
        assert np.array_equal(keys.cpu().numpy(), want), (sweep, seed)
    print(f"PARITY sample_order n={n} chains={chains} chain0={chain0}: bit-identical to the numpy restatement")


# ---- 2. the token-set sampler ---------------------------------------------------------------------------------------
SETS = {1: [7], 20: AA, 21: AA + [GAP], 32: [int(v) for v in np.random.default_rng(32).permutation(33)[:32]]}


@pytest.mark.parametrize("tau", [0.05, 1.0, 20.0])
@pytest.mark.parametrize("n_set", sorted(SETS))
@pytest.mark.parametrize("per", [1, 7, 40])
def test_sample_rows_over_token_sets_against_float64(per, n_set, tau):
    from esm_b200 import variants
    token_set = SETS[n_set]
    R, C, chains = 5, 9, 6  # 40 entries per alignment
    W = C - 1
    n = chains * per
    g = torch.Generator(device="cuda").manual_seed(per * 1000 + n_set * 10 + int(tau))
    logits = torch.randn((n, 33), device="cuda", generator=g) * 3
    ent = torch.stack([torch.randperm(R * W, device="cuda", generator=g)[:per] for _ in range(chains)]).view(-1)
    tokens = torch.randint(0, 33, (chains, R, C), device="cuda", generator=g)
    before = tokens.clone()
    seed, step, chain0 = 2 ** 64 - 5, 11, 2 ** 32 - chains
    logp = torch.full((chains, 3), float("nan"), device="cuda")
    logq = _rows(logits, token_set, tau, seed, step, chain0, per, ent, tokens, R, C, logp[:, 1], 3)
    z = _tempered(logits[:, token_set], tau)
    chain = chain0 + np.arange(n) // per
    entries = ent.cpu().numpy()
    score, want = sr.draw_f64(z.cpu().numpy(), step, chain, entries, seed)
    r, j = sr.entry_token(entries, C)
    local = np.arange(n) // per
    got_tok = tokens.cpu().numpy()[local, r, j]
    lookup = {t: a for a, t in enumerate(token_set)}
    got = np.array([lookup.get(int(t), -1) for t in got_tok])
    close = sr.top_two_gap(score) <= NEAR_TIE if n_set > 1 else np.zeros(n, dtype=bool)
    mism = int((got != want)[~close].sum())
    print(f"PARITY sample_rows |A|={n_set} per={per} tau={tau}: {mism} draws differ from float64 away from "
          f"near-ties, {int(close.sum())} near-ties")
    assert mism == 0 and bool((got >= 0).all())
    ref = variants.log_softmax_rows(z.contiguous(), torch.as_tensor(got, device="cuda"))
    assert torch.equal(logq, ref), "logq must equal esmb200_log_softmax_rows bit for bit"
    changed = (tokens != before).cpu().numpy()
    targeted = np.zeros_like(changed)
    targeted[local, r, j] = True
    assert not (changed & ~targeted).any(), "only the targeted entries may change"
    lq = logq.view(chains, per).cpu().numpy()
    acc = np.zeros(chains, dtype=np.float32)
    for k in range(per):
        acc = acc + lq[:, k]
    assert np.array_equal(logp[:, 1].cpu().numpy(), acc)
    assert bool(logp[:, 0].isnan().all()) and bool(logp[:, 2].isnan().all())


@pytest.mark.parametrize("n_set", [20, 21, 32])
def test_sample_rows_ties_go_to_the_smaller_index_and_out_of_range_entries_write_nothing(n_set):
    """Two set members at 1e30 and the rest at -1e30: every Gumbel score rounds to 1e30 exactly, a tie, so the
    smaller index wins with log q = -log 2. Entries -1 and R (C - 1) write nothing and give a NaN log q."""
    token_set = SETS[n_set]
    R, C = 3, 6
    pairs = [(0, 1), (2, n_set - 1), (n_set - 2, n_set - 1), (5, 9)]
    logits = torch.full((len(pairs) + 2, 33), -1e30, device="cuda")
    for i, (a, b) in enumerate(pairs):
        logits[i, token_set[a]] = logits[i, token_set[b]] = 1e30
    ent = torch.tensor([0, 4, 9, 14, -1, R * (C - 1)], device="cuda")
    tokens = torch.zeros((6, R, C), dtype=torch.int64, device="cuda")
    logq = _rows(logits, token_set, 1.0, 3, 0, 0, 1, ent, tokens, R, C)
    for i, (a, _) in enumerate(pairs):
        r, j = sr.entry_token(int(ent[i]), C)
        assert int(tokens[i, r, j]) == token_set[a], (i, a)
        assert float(logq[i]) == pytest.approx(-np.log(2), abs=1e-6)
    assert bool(logq[-2:].isnan().all()) and int(tokens[-2:].abs().sum()) == 0
    assert int((tokens != 0).sum()) == len(pairs)
    print(f"PARITY sample_rows |A|={n_set}: ties to the smaller index, out-of-range entries write nothing")


# ---- 3. statistics ----------------------------------------------------------------------------------------------------
def test_two_hundred_thousand_draws_over_21_tokens_follow_the_tempered_softmax():
    from scipy.stats import chisquare
    token_set = AA + [GAP]
    z = torch.linspace(-3.0, 1.0, 21)
    tau = 0.8
    logits = torch.zeros((25000, 33), device="cuda")
    logits[:, token_set] = z.cuda()
    ent = torch.zeros(25000, dtype=torch.int64, device="cuda")
    counts = torch.zeros(33, dtype=torch.int64)
    for step in range(8):  # 8 steps x 25,000 chains
        tokens = torch.zeros((25000, 1, 2), dtype=torch.int64, device="cuda")
        _rows(logits, token_set, tau, 31337, step, 0, 1, ent, tokens, 1, 2)
        counts += torch.bincount(tokens[:, 0, 1].cpu(), minlength=33)
    assert int(counts.sum()) == 200000 and int(counts[token_set].sum()) == 200000
    p = torch.softmax(_tempered(z, tau).double(), 0).numpy()
    stat, pval = chisquare(counts[token_set].numpy(), p * 200000)
    print(f"PARITY sample_rows chi-square of 200,000 draws over 21 tokens: {stat:.2f} on 20 dof, p = {pval:.3g}")
    assert pval > 1e-3


# ---- 4. msa_gibbs on the tiny MSA fixture ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def msa_fixture(golden_dir):
    import variant_fixtures as vf
    from esm_b200 import pretrained, variants
    with open(os.path.join(golden_dir, "variants.json")) as f:
        a3m = json.load(f)["a3m"]
    with tempfile.TemporaryDirectory() as tmp:
        path = vf.write_checkpoint("msa_t2_tiny", vf.MODELS["msa_t2_tiny"], tmp)
        model, alphabet = pretrained.load_msa_model_and_alphabet(path)
        with open(os.path.join(tmp, "in.a3m"), "w") as f:
            f.write(a3m)
        msa = variants.read_msa(os.path.join(tmp, "in.a3m"), 7)
    tokens = alphabet.get_batch_converter()(msa)[2]
    return model.eval().cuda(), alphabet, tokens.cuda(), msa, a3m


def _with_appended(model, tokens, k):
    new = torch.full((1, k, tokens.shape[2]), model.mask_idx, dtype=torch.int64, device=tokens.device)
    new[:, :, 0] = model.cls_idx
    return torch.cat([tokens, new], 1)


def _designable(R, W, appended, seed=0):
    g = torch.Generator().manual_seed(seed)
    des = torch.rand((R, W), generator=g) < 0.08
    des[R - appended:] = True
    return des


@pytest.mark.parametrize("precision", ["fp16", "fp32x3"])
def test_msa_gibbs_on_the_tiny_fixture(msa_fixture, precision):
    from esm_b200 import sampling
    model, _, tokens, _, _ = msa_fixture
    model.set_precision(precision)
    try:
        x = _with_appended(model, tokens, 2)
        R, C = x.shape[1:]
        des = _designable(R, C - 1, 2).cuda()
        kw = dict(designable=des, chains=4, sweeps=2, block=9, temperature=0.7, seed=2 ** 40 + 3)
        a = sampling.msa_gibbs(model, x, **kw)
        t, lp = a["tokens"], a["logp"]
        n = int(des.sum())
        steps = 2 * -(-n // 9)
        assert t.shape == (4, R, C) and t.dtype == torch.int64 and lp.shape == (4, steps) and lp.dtype == torch.float32
        assert bool(lp.isfinite().all()) and bool((lp <= 0).all())
        full = torch.zeros((R, C), dtype=torch.bool, device="cuda")
        full[:, 1:] = des
        assert torch.equal(t[:, ~full], x[0][~full].expand(4, -1)), "fixed entries and <cls> never change"
        drawable = torch.tensor(AA + [GAP], device="cuda")
        assert bool(torch.isin(t[:, full], drawable).all())
        # one sweep from the appended <mask> rows leaves no <mask>; without gaps only amino acids are drawn
        one = sampling.msa_gibbs(model, x, **{**kw, "sweeps": 1, "gaps": False})
        assert not bool((one["tokens"] == model.mask_idx).any())
        assert bool(torch.isin(one["tokens"][:, full], drawable[:20]).all())
        # the same bits for every chunk size and for repeated calls; another seed differs
        for max_tokens in (R * C, 3 * R * C, 1):
            b = sampling.msa_gibbs(model, x, max_tokens=max_tokens, **kw)
            assert torch.equal(a["tokens"], b["tokens"]) and torch.equal(a["logp"], b["logp"]), max_tokens
        b = sampling.msa_gibbs(model, x, **kw)
        assert torch.equal(a["tokens"], b["tokens"]) and torch.equal(a["logp"], b["logp"])
        d = sampling.msa_gibbs(model, x, **{**kw, "seed": 4})
        assert not torch.equal(a["tokens"], d["tokens"])
        print(f"PARITY msa_gibbs msa_t2_tiny {precision}: fixed entries kept, drawable tokens only, no <mask> after "
              f"sweep 0, chunking and repeats bit-identical")
    finally:
        model.set_precision("fp16")


@pytest.mark.parametrize("gaps", [True, False])
@pytest.mark.parametrize("precision", ["fp16", "fp32x3"])
def test_every_step_replayed_through_the_public_forward(msa_fixture, precision, gaps):
    """Each chain replayed one step at a time: the restated order, the block masked, model(masked)["logits"] at the
    block's entries, the float64 Gumbel draw on those logits and esmb200_log_softmax_rows for log q. Tokens and logp
    must equal msa_gibbs' bit for bit (no step of this seed has a near-tie)."""
    from esm_b200 import sampling, variants
    model, _, tokens, _, _ = msa_fixture
    model.set_precision(precision)
    try:
        x = _with_appended(model, tokens, 1)
        R, C = x.shape[1:]
        des = _designable(R, C - 1, 1, seed=1)
        entries = des.view(-1).nonzero().view(-1).numpy()
        tau, seed, sweeps, block, chains = 1.3, 2024, 2, 11, 2
        out = sampling.msa_gibbs(model, x, designable=des, chains=chains, sweeps=sweeps, block=block,
                                 temperature=tau, seed=seed, gaps=gaps)
        token_set = AA + [GAP] if gaps else AA
        min_gap = np.inf
        for c in range(chains):
            state = x.clone()
            s = 0
            logp = []
            for w in range(sweeps):
                for blk in sr.sweep_blocks(entries, c, w, seed, block):
                    r, j = sr.entry_token(blk, C)
                    masked = state.clone()
                    masked[0, r, j] = model.mask_idx
                    logits = model(masked)["logits"][0, r, j][:, token_set].float()
                    z = _tempered(logits, tau)
                    score, a = sr.draw_f64(z.cpu().numpy(), s, np.full(len(blk), c), blk, seed)
                    min_gap = min(min_gap, float(sr.top_two_gap(score).min()))
                    logq = variants.log_softmax_rows(z.contiguous(), torch.as_tensor(a, device="cuda")).cpu().numpy()
                    acc = np.float32(0)
                    for v in logq:
                        acc = np.float32(acc + v)
                    logp.append(acc)
                    state[0, r, j] = torch.tensor(token_set, device="cuda")[torch.as_tensor(a, device="cuda")]
                    s += 1
            assert torch.equal(out["tokens"][c], state[0]), c
            assert np.array_equal(out["logp"][c].cpu().numpy(), np.array(logp, dtype=np.float32)), c
        print(f"PARITY msa_gibbs replay {precision} gaps={gaps}: {chains} chains x {s} steps through the public "
              f"forward, tokens and logp bit-identical; smallest top-two Gumbel gap {min_gap:.3g}")
        assert min_gap > NEAR_TIE
    finally:
        model.set_precision("fp16")


# ---- 5. against the float64 oracle ------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision,tol", [("fp16", 2e-2), ("fp32x3", 1e-3)])
def test_one_step_against_the_float64_oracle(msa_fixture, precision, tol):
    """One step (block = every designable entry): the logits at the block's entries against msa_transformer_forward
    in float64, centred rel-Frobenius over the vocabulary; the draws must agree wherever the oracle's top-two Gumbel
    gap exceeds twice the row's largest tempered-logit error."""
    import variant_fixtures as vf
    from esm_b200 import sampling
    from oracle.msa_oracle import msa_transformer_forward
    model, _, tokens, _, _ = msa_fixture
    cfg = vf.MODELS["msa_t2_tiny"]
    sd = {k: v.double() for k, v in vf.state_dict(cfg).items()}
    model.set_precision(precision)
    try:
        x = _with_appended(model, tokens, 1)
        R, C = x.shape[1:]
        des = _designable(R, C - 1, 1, seed=2)
        entries = des.view(-1).nonzero().view(-1).numpy()
        tau, seed, chains = 0.9, 55, 3
        out = sampling.msa_gibbs(model, x, designable=des, chains=chains, block=len(entries), temperature=tau,
                                 seed=seed)
        blk = sr.sweep_blocks(entries, 0, 0, seed, len(entries))[0]
        r, j = sr.entry_token(blk, C)
        masked = x.clone()
        masked[0, r, j] = model.mask_idx
        got = model(masked)["logits"][0, r, j].double().cpu()
        want = msa_transformer_forward(sd, cfg["layers"], cfg["attention_heads"], masked.cpu())["logits"][0, r, j]
        gc, wc = got - got.mean(-1, keepdim=True), want - want.mean(-1, keepdim=True)
        rel = float((gc - wc).norm() / wc.norm())
        token_set = AA + [GAP]
        z_ref = want[:, token_set].numpy() / np.float32(tau)
        err = np.abs(_tempered(got[:, token_set].float().cuda(), tau).double().cpu().numpy() - z_ref).max(-1)
        agree, decided = 0, 0
        for c in range(chains):
            score, a = sr.draw_f64(z_ref, 0, np.full(len(blk), c), blk, seed)
            sure = sr.top_two_gap(score) > 2 * err
            drawn = out["tokens"][c, r, j].cpu().numpy()
            decided += int(sure.sum())
            agree += int((drawn == np.array(token_set)[a])[sure].sum())
        print(f"PARITY msa_gibbs one step {precision} vs float64 oracle: centred rel_fro {rel:.2e} (tol {tol}); "
              f"{agree}/{decided} decided draws agree")
        assert rel <= tol
        assert decided > 0 and agree == decided
    finally:
        model.set_precision("fp16")


# ---- 6. host synchronisation ------------------------------------------------------------------------------------------
def test_no_host_synchronisation_after_the_first_step(msa_fixture):
    from esm_b200 import sampling
    model, _, tokens, _, _ = msa_fixture
    x = _with_appended(model, tokens, 2)
    R, C = x.shape[1:]
    stack = model._stack_unpadded
    calls = []

    def first_then_strict(*args, **kwargs):
        out = stack(*args, **kwargs)
        if not calls:
            torch.cuda.set_sync_debug_mode("error")  # every later step, sweep and chunk must not synchronise
        calls.append(1)
        return out

    model._stack_unpadded = first_then_strict
    try:
        des = _designable(R, C - 1, 2, seed=3)
        n = int(des.sum())
        out = sampling.msa_gibbs(model, x, designable=des, chains=6, sweeps=3, block=20, seed=1,
                                 max_tokens=3 * R * C)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        del model._stack_unpadded
    assert len(calls) == 2 * 3 * -(-n // 20)  # 2 chunks x 3 sweeps x blocks
    assert not bool((out["tokens"] == model.mask_idx).any())


# ---- 7. the command line ----------------------------------------------------------------------------------------------
def test_cli_end_to_end(msa_fixture, tmp_path):
    import variant_fixtures as vf
    from esm_b200 import sample_msa_cli, sampling, variants
    model, alphabet, tokens, msa, a3m = msa_fixture
    path = vf.write_checkpoint("msa_t2_tiny", vf.MODELS["msa_t2_tiny"], str(tmp_path))
    (tmp_path / "in.a3m").write_text(a3m)
    out = tmp_path / "out"
    argv = [path, "--msa", str(tmp_path / "in.a3m"), "--msa-samples", "5", "--rows", "1", "--columns", "3-6,40",
            "--append-rows", "2", "--chains", "3", "--sweeps", "2", "--block", "7", "--temperature", "0.9",
            "--seed", "9", "--max-tokens", "200", "--out", str(out)]
    assert sample_msa_cli.run(sample_msa_cli.create_parser().parse_args(argv)) == 3
    x = _with_appended(model, tokens[:, :5], 2)
    R, C = x.shape[1:]
    des = sample_msa_cli.designable_mask(5, C - 1, 2, [0], [2, 3, 4, 5, 39])
    want = sampling.msa_gibbs(model, x, designable=des, chains=3, sweeps=2, block=7, temperature=0.9, seed=9)
    names = [d for d, _ in msa[:5]] + ["generated_0", "generated_1"]
    per_sweep = want["logp"].shape[1] // 2
    rows = (out / "samples.tsv").read_text().splitlines()
    assert rows[0] == "chain\tseed\tlogp" and len(rows) == 4
    for c in range(3):
        back = variants.read_msa(out / f"sample_{c}.a3m", 100)
        assert [d for d, _ in back] == names
        seqs = [s for _, s in back]
        assert seqs == ["".join(alphabet.get_tok(int(t)) for t in row[1:]) for row in want["tokens"][c]]
        for r in range(5):  # fixed entries are the input's
            assert all(seqs[r][k] == msa[r][1][k] for k in range(C - 1) if not des[r, k])
        assert "<mask>" not in "".join(seqs)
        lp = float(want["logp"][c, -per_sweep:].double().sum())
        assert rows[1 + c] == f"{c}\t9\t{lp:.4f}"
    print("PARITY sample_msa_cli: a3m files and samples.tsv equal the API's samples, fixed entries kept")
