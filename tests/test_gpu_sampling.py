"""GPU: Gibbs sampling of sequences (esm_b200.sampling.gibbs, esmb200_sample_order, esmb200_sample_rows).

  1. the sampler kernel in the sequence layout (the 20 amino acids, R = 1, C = T - 1, stride T) against the
     float64/numpy oracle at several temperatures and row counts: a* on every row
     whose top two scores are more than 1e-5 apart, log q bit for bit against esmb200_log_softmax_rows, only the
     targeted token entries written, the block sums of log q;
  2. the order kernel on residue indices against the numpy restatement, bit for bit;
  3. a chi-square test of 200,000 draws of one row against softmax(z);
  4. tiny ESM-2 and ESM-1b models in fp16, fp32x3 and fp8: fixed positions, amino acids only after sweep 0 of a de novo
     start, reproducibility, chunking, log q against the public forward, the tokens against the oracle's draw;
  5. cpu_offload() bit-identical; no host synchronisation after the first step;
  6. the command line end to end.
Every gated comparison prints a PARITY line.
"""
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

AA0 = 4  # AMINO_ACIDS are tokens 4 ... 23 of the ESM-1b / ESM-2 alphabet
AA = list(range(AA0, AA0 + 20))
NEAR_TIE = 1e-5


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _rows(logits, tau, seed, step, chain0, per, pos, tokens, logp=None, stride=0):
    """esmb200_sample_rows in the sequence layout: the 20 amino acids, tokens [chains, T] as R = 1, C = T - 1."""
    from esm_b200 import _lib
    n = logits.shape[0]
    T = tokens.shape[1]
    ts = torch.tensor(AA, dtype=torch.int32, device="cuda")
    logq = torch.full((n,), float("nan"), device="cuda")
    rc = _lib.load().esmb200_sample_rows(logits.data_ptr(), logits.stride(0), n, ts.data_ptr(), len(AA), tau, seed,
                                         step, chain0, per, pos.data_ptr(), tokens.data_ptr(), T, 1, T - 1,
                                         logq.data_ptr(), logp.data_ptr() if logp is not None else None, stride,
                                         _stream())
    _lib.check(rc)
    return logq


def _tempered(logits, tau):
    """logits / fp32(tau) by IEEE fp32 division, as the kernel divides. (A CUDA tensor divided by a Python number is
    multiplied by the reciprocal instead, which differs in the last bit.)"""
    return logits / torch.full_like(logits, tau)


# ---- 1. the sampler kernel ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tau", [0.3, 1.0, 2.5])
@pytest.mark.parametrize("n,per", [(1, 1), (31, 31), (32, 4), (65537, 1)])
def test_sample_rows_in_the_sequence_layout_against_float64(n, per, tau):
    from esm_b200 import variants
    g = torch.Generator(device="cuda").manual_seed(n * 7 + int(tau * 10))
    T = 300
    chains = n // per
    logits = torch.randn((n, 33), device="cuda", generator=g) * 3
    pos = torch.stack([torch.randperm(T - 2, device="cuda", generator=g)[:per] for _ in range(chains)]).view(-1)
    tokens = torch.randint(0, 33, (chains, T), device="cuda", generator=g)
    before = tokens.clone()
    seed, step, chain0 = 2 ** 64 - 5, 11, 7
    logp = torch.full((chains, 3), float("nan"), device="cuda")
    logq = _rows(logits, tau, seed, step, chain0, per, pos, tokens, logp[:, 1], 3)
    z = _tempered(logits[:, AA0:AA0 + 20], tau)
    chain = chain0 + np.arange(n) // per
    score, want = sr.draw_f64(z.cpu().numpy(), step, chain, pos.cpu().numpy(), seed)
    rows = torch.arange(n, device="cuda") // per
    got = (tokens[rows, pos + 1] - AA0).cpu().numpy()
    close = sr.top_two_gap(score) <= NEAR_TIE
    mism = int((got != want)[~close].sum())
    print(f"PARITY sample_rows n={n} tau={tau}: {mism} draws differ from float64 away from near-ties, {int(close.sum())} "
          f"rows have top two scores within {NEAR_TIE}")
    assert mism == 0 and bool(((got >= 0) & (got < 20)).all())
    ref = variants.log_softmax_rows(z.contiguous(), torch.as_tensor(got, device="cuda"))
    assert torch.equal(logq, ref), "logq must equal esmb200_log_softmax_rows bit for bit"
    changed = tokens != before
    targeted = torch.zeros_like(changed)
    targeted[rows, pos + 1] = True
    assert not bool((changed & ~targeted).any()), "only the targeted entries may change"
    lq = logq.view(chains, per).cpu().numpy()
    acc = np.zeros(chains, dtype=np.float32)
    for j in range(per):
        acc = acc + lq[:, j]
    assert np.array_equal(logp[:, 1].cpu().numpy(), acc)
    assert bool(logp[:, 0].isnan().all()) and bool(logp[:, 2].isnan().all())


def test_sequence_layout_argument_checks_and_an_out_of_range_position():
    from esm_b200 import _lib
    logits = torch.zeros((2, 33), device="cuda")
    tokens = torch.zeros((2, 6), dtype=torch.int64, device="cuda")
    pos = torch.tensor([3, 4], device="cuda")  # 4 = T - 2: outside [0, T - 2)
    logq = _rows(logits, 1.0, 0, 0, 0, 1, pos, tokens)
    assert bool(logq[1].isnan()) and int(tokens[1].abs().sum()) == 0
    assert AA0 <= int(tokens[0, 4]) < AA0 + 20 and float(logq[0]) == pytest.approx(-np.log(20), abs=1e-6)
    ts = torch.tensor(AA, dtype=torch.int32, device="cuda")
    assert _lib.load().esmb200_sample_rows(logits.data_ptr(), 33, 2, ts.data_ptr(), 20, 0.0, 0, 0, 0, 1, pos.data_ptr(),
                                           tokens.data_ptr(), 6, 1, 5, logq.data_ptr(), None, 0, _stream()) == -1


# ---- 2. the order kernel --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,chains,chain0", [(1, 1, 0), (37, 5, 2 ** 32 - 5), (1022, 64, 3)])
def test_sample_order_of_residue_indices_matches_the_restatement(n, chains, chain0):
    from esm_b200 import _lib
    g = np.random.default_rng(n)
    positions = g.choice(65535, n, replace=False)
    positions[0] = 65534
    pos = torch.as_tensor(positions, device="cuda")
    keys = torch.empty((chains, n), dtype=torch.int64, device="cuda")
    for sweep, seed in [(0, 0), (9, 2 ** 64 - 1)]:
        _lib.check(_lib.load().esmb200_sample_order(pos.data_ptr(), n, chains, chain0, sweep, seed, keys.data_ptr(),
                                                    _stream()))
        want = sr.order_keys(positions, chain0 + np.arange(chains), sweep, seed)
        assert np.array_equal(keys.cpu().numpy(), want), (sweep, seed)
    print(f"PARITY sample_order n={n} chains={chains}: bit-identical to the numpy restatement")


# ---- 3. statistics ----------------------------------------------------------------------------------------------------
def test_two_hundred_thousand_sequence_layout_draws_follow_softmax():
    from scipy.stats import chisquare
    z = torch.linspace(-3.0, 1.0, 20)
    logits = torch.zeros((25000, 33), device="cuda")
    logits[:, AA0:AA0 + 20] = z.cuda()
    pos = torch.zeros(25000, dtype=torch.int64, device="cuda")
    counts = torch.zeros(20, dtype=torch.int64)
    for step in range(8):  # 8 steps x 25,000 chains
        tokens = torch.zeros((25000, 3), dtype=torch.int64, device="cuda")
        _rows(logits, 1.0, 31337, step, 0, 1, pos, tokens)
        counts += torch.bincount((tokens[:, 1] - AA0).cpu(), minlength=20)
    p = torch.softmax(z.double(), 0).numpy()
    stat, pval = chisquare(counts.numpy(), p * 200000)
    print(f"PARITY sample_rows chi-square of 200,000 draws: {stat:.2f} on 19 dof, p = {pval:.3g}")
    assert pval > 1e-3


# ---- 4. models ------------------------------------------------------------------------------------------------------
def _fixture_model(name, tmp):
    import variant_fixtures as vf
    from esm_b200 import pretrained
    model, alphabet = pretrained.load_model_and_alphabet(vf.write_checkpoint(name, vf.MODELS[name], tmp))
    return model.eval().cuda(), alphabet


@pytest.fixture(scope="module")
def fixtures():
    with tempfile.TemporaryDirectory() as tmp:
        yield {n: _fixture_model(n, tmp) for n in ("esm2_t2_tiny", "esm1b_t2_tiny")}


def _start(alphabet, seq):
    return alphabet.get_batch_converter()([("p", seq)])[2].cuda()


def _de_novo(model, L):
    return torch.tensor([[model.cls_idx] + [model.mask_idx] * L + [model.eos_idx]], device="cuda")


@pytest.mark.parametrize("precision", ["fp16", "fp32x3", "fp8"])
@pytest.mark.parametrize("name", ["esm2_t2_tiny", "esm1b_t2_tiny"])
def test_gibbs_on_a_tiny_model(fixtures, name, precision):
    from esm_b200 import sampling
    model, alphabet = fixtures[name]
    model.set_precision(precision)
    try:
        # de novo: every designable position holds an amino acid after sweep 0
        x0 = _de_novo(model, 30)
        out = sampling.gibbs(model, x0, chains=3, sweeps=1, block=4, seed=5)
        t, lp = out["tokens"], out["logp"]
        assert t.shape == (3, 32) and t.dtype == torch.int64 and lp.shape == (3, 8) and lp.dtype == torch.float32
        assert bool(((t[:, 1:-1] >= AA0) & (t[:, 1:-1] < AA0 + 20)).all())
        assert bool((t[:, 0] == model.cls_idx).all()) and bool((t[:, -1] == model.eos_idx).all())
        assert bool(lp.isfinite().all()) and bool((lp <= 0).all())
        # fixed positions unchanged; same seed same bits, another seed not; one chain per chunk equals one chunk
        seq = "MKTAYIAKQRQISFVKSHFSRQLEERLGLIEVQ"
        x = _start(alphabet, seq)
        D = [0, 3, 4, 5, 10, 11, 20, 31]
        kw = dict(positions=D, chains=4, sweeps=3, block=3, temperature=0.7, seed=2 ** 40 + 3)
        a = sampling.gibbs(model, x, **kw)
        fixed = [i for i in range(len(seq)) if i not in D]
        assert torch.equal(a["tokens"][:, [1 + i for i in fixed]], x[:, [1 + i for i in fixed]].expand(4, -1))
        assert a["logp"].shape == (4, 9)
        b = sampling.gibbs(model, x, **kw)
        assert torch.equal(a["tokens"], b["tokens"]) and torch.equal(a["logp"], b["logp"])
        c = sampling.gibbs(model, x, max_tokens=x.shape[1], **kw)
        assert torch.equal(a["tokens"], c["tokens"]) and torch.equal(a["logp"], c["logp"])
        d = sampling.gibbs(model, x, **{**kw, "seed": 4})
        assert not torch.equal(a["tokens"], d["tokens"])
        # chunks of 3 and 1 chains
        e = sampling.gibbs(model, x, max_tokens=3 * x.shape[1], **kw)
        assert torch.equal(a["tokens"], e["tokens"])
        print(f"PARITY gibbs {name} {precision}: de novo all amino acids, fixed positions kept, reproducible, "
              f"chunking bit-identical")
    finally:
        model.set_precision("fp16")


@pytest.mark.parametrize("precision", ["fp16", "fp32x3", "fp8"])
@pytest.mark.parametrize("name", ["esm2_t2_tiny", "esm1b_t2_tiny"])
def test_one_step_against_the_public_forward_and_the_oracle(fixtures, name, precision):
    """block = |D|, one sweep: one step. Its logp equals log_softmax(model(x_masked)["logits"][rows][:, AA] / tau) at
    the drawn tokens, and the tokens are the oracle's Gumbel-max draw on those logits, except at near-ties."""
    from esm_b200 import sampling
    model, alphabet = fixtures[name]
    model.set_precision(precision)
    try:
        seq = "MKTAYIAKQRQISFVKSHFSRQLEERLGLIEVQAPILSRVGDGTQDNLSGAEKAVQ"
        x = _start(alphabet, seq)
        D = [1, 2, 9, 17, 30, 44, 45, 52]
        tau, seed, C = 0.8, 77, 6
        out = sampling.gibbs(model, x, positions=D, chains=C, block=len(D), temperature=tau, seed=seed)
        assert out["logp"].shape == (C, 1)
        xm = x.clone()
        xm[0, [1 + p for p in D]] = model.mask_idx  # built on the host side of the API: the public forward
        logits = model(xm)["logits"][0, [1 + p for p in D]][:, AA0:AA0 + 20]
        z = _tempered(logits, tau)
        lsm = torch.log_softmax(z.double(), -1)
        drawn = out["tokens"][:, [1 + p for p in D]] - AA0
        want_logp = lsm.gather(1, drawn.T).sum(0)  # [C]: sum over the block of log q of each chain's draws
        err = float((out["logp"][:, 0].double() - want_logp).abs().max())
        zn = z.float().cpu().numpy()
        mism, ties = 0, 0
        for c in range(C):
            score, want = sr.draw_f64(zn, 0, np.full(len(D), c), np.array(D), seed)
            close = sr.top_two_gap(score) <= NEAR_TIE
            ties += int(close.sum())
            mism += int((drawn[c].cpu().numpy() != want)[~close].sum())
        print(f"PARITY gibbs one step {name} {precision}: max |logp - log_softmax(public forward)| = {err:.2e}, "
              f"{mism} draws differ from the oracle away from near-ties, {ties} near-ties")
        assert err <= 1e-5 * len(D)
        assert mism == 0
    finally:
        model.set_precision("fp16")


# ---- 5. cpu_offload() and host synchronisation ----------------------------------------------------------------------
def test_cpu_offload_is_bit_identical(tmp_path):
    from esm_b200 import sampling
    model, alphabet = _fixture_model("esm1b_t2_tiny", str(tmp_path))
    x = _start(alphabet, "MKTAYIAKQRQISFVKSHFSRQLEERLGLIEVQ")
    kw = dict(positions=list(range(4, 20)), chains=5, sweeps=2, block=5, temperature=1.3, seed=123)
    want = sampling.gibbs(model, x, **kw)
    model.cpu_offload()
    try:
        got = sampling.gibbs(model, x, max_tokens=2 * x.shape[1], **kw)
    finally:
        model.cuda()
    print("PARITY gibbs esm1b_t2_tiny cpu_offload(): tokens and logp bit-identical to resident")
    assert torch.equal(got["tokens"], want["tokens"]) and torch.equal(got["logp"], want["logp"])


def test_no_host_synchronisation_after_the_first_step(fixtures):
    from esm_b200 import sampling
    model, _ = fixtures["esm2_t2_tiny"]
    stack = model._stack
    calls = []

    def first_then_strict(*args, **kwargs):
        out = stack(*args, **kwargs)
        if not calls:
            torch.cuda.set_sync_debug_mode("error")  # every later step, sweep and chunk must not synchronise
        calls.append(1)
        return out

    model._stack = first_then_strict
    try:
        out = sampling.gibbs(model, _de_novo(model, 40), chains=6, sweeps=3, block=7, seed=1, max_tokens=3 * 42)
    finally:
        torch.cuda.set_sync_debug_mode(0)
        del model._stack
    assert len(calls) == 2 * 3 * 6  # 2 chunks x 3 sweeps x 6 blocks
    assert bool(((out["tokens"][:, 1:-1] >= AA0) & (out["tokens"][:, 1:-1] < AA0 + 20)).all())


# ---- 6. the command line ----------------------------------------------------------------------------------------------
def test_cli_end_to_end(tmp_path):
    import variant_fixtures as vf
    from esm_b200 import pretrained, sample_cli, sampling
    path = vf.write_checkpoint("esm2_t2_tiny", vf.MODELS["esm2_t2_tiny"], str(tmp_path))
    model, alphabet = pretrained.load_model_and_alphabet(path)
    model = model.eval().cuda()
    runs = [(["--length", "24", "--chains", "3", "--sweeps", "2", "--block", "5", "--seed", "9"],
             _de_novo(model, 24), dict(chains=3, sweeps=2, block=5, seed=9)),
            (["--sequence", "MKTAYIAKQRQISFVK", "--positions", "2-5,9", "--chains", "2", "--temperature", "0.5",
              "--max-tokens", "18"],
             _start(alphabet, "MKTAYIAKQRQISFVK"), dict(positions=[1, 2, 3, 4, 8], chains=2, temperature=0.5))]
    for k, (argv, x, kw) in enumerate(runs):
        fasta = tmp_path / f"s{k}.fasta"
        args = sample_cli.create_parser().parse_args([path, *argv, "--out", str(fasta)])
        assert sample_cli.run(args) == kw["chains"]
        want = sampling.gibbs(model, x, **kw)
        lines = fasta.read_text().splitlines()
        assert len(lines) == 2 * kw["chains"]
        per_sweep = want["logp"].shape[1] // kw.get("sweeps", 1)
        for c in range(kw["chains"]):
            lp = float(want["logp"][c, -per_sweep:].double().sum())
            assert lines[2 * c] == f">sample_{c} seed={kw.get('seed', 0)} logp={lp:.4f}"
            assert lines[2 * c + 1] == "".join(alphabet.get_tok(int(t)) for t in want["tokens"][c, 1:-1])
    print("PARITY sample_cli: FASTA records equal the API's samples")
