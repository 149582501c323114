"""GPU: variant-effect scoring (esm_b200.variants, esm_b200.predict_cli) against the reference's
examples/variant-prediction/predict.py.

  * esmb200_log_softmax_rows against torch.log_softmax;
  * every (model, strategy) of tests/golden/variants.json (predict.py's own output tables, CPU fp32) at DESIGN.md
    section 4's logits tolerances, and fp32x3 at least 10x closer than fp16;
  * batching is exact: masked_marginals does not depend on the chunk size and equals a loop of model(...)["logits"]
    through the same kernel; pseudo_ppl batched across mutants equals one mutant at a time;
  * full size against the unmodified reference (oracle/_ref) running predict.py's batch-1 loop, eager fp32;
  * model.half(), and the command line end to end.
"""
import argparse
import csv
import io
import json
import math
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # variant_fixtures, esm1b_weights

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")
REL_FRO = 4e-3      # DESIGN.md section 4, logits
MAX_ABS_RMS = 2e-2  # max-abs error over the rms of the reference scores
BLAT_ECOLX = ("HPETLVKVKDAEDQLGARVGYIELDLNSGKILESFRPEERFPMMSTFKVLLCGAVLSRVDAGQEQLGRRIHYSQNDLVEYSPVTEKHLTDGMTVRELCSAAIT"
              "MSDNTAANLLLTTIGGPKELTAFLHNMGDHVTRLDRWEPELNEAIPNDERDTTMPAAMATTLRKLLTGELLTLASRQQLIDWMEADKVAGPLLRSALPAGWFIA"
              "DKSGAGERGSRGIIAALGPDGKPSRIVVIYTTGSQATMDERNRQIAEIGASLIKHW")  # examples/variant-prediction/README.md:12


def rel_fro(a, b):
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    return float((a - b).norm() / b.norm())


@pytest.fixture(scope="module")
def fixture(golden_dir):
    with open(os.path.join(golden_dir, "variants.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def esm_ref():
    if not os.path.isdir(os.path.join(REF, "esm")):
        pytest.fail("oracle/_ref/esm is missing: build() copies the reference there (oracle/reference.py)")
    sys.path.insert(0, REF)
    try:
        import esm  # the reference
        yield esm
    finally:
        sys.path.remove(REF)


def fixture_model(fixture, name, precision="fp16"):
    """The fixture model loaded the way predict.py loads it: from its checkpoint (the ESM-1b loader zeroes the <mask>
    row of the tied embedding, which the log-softmax normaliser sees)."""
    import tempfile
    import variant_fixtures as vf
    from esm_b200 import predict_cli
    cfg = fixture["models"][name]
    assert abs(vf.checksum(vf.state_dict(cfg)) - cfg["state_dict_checksum"]) <= 1e-6 * cfg["state_dict_checksum"]
    with tempfile.TemporaryDirectory() as tmp:
        model = predict_cli.load_model(vf.write_checkpoint(name, cfg, tmp))[0]
    model = model.cuda()
    if precision != "fp16":
        model.set_precision(precision)
    return model


def reference_table(fixture, name, strategy):
    table = list(csv.reader(io.StringIO(fixture["outputs"][f"{name}/{strategy}"])))
    return table, [float(r[-1]) for r in table[1:]]


def cli_args(fixture, strategy, tmp_path, max_tokens=None):
    from esm_b200 import variants
    msa = tmp_path / "msa.a3m"
    msa.write_text(fixture["a3m"])
    return argparse.Namespace(sequence=fixture["sequence"], offset_idx=fixture["offset_idx"], scoring_strategy=strategy,
                              msa_path=msa, msa_samples=fixture["msa_samples"],
                              max_tokens=max_tokens or variants.DEFAULT_MAX_TOKENS)


def mutations(fixture):
    return [r[0] for r in list(csv.reader(io.StringIO(fixture["dms_csv"])))[1:]]


CASES = [(n, s) for n in ("esm2_t2_tiny", "esm1b_t2_tiny") for s in ("wt-marginals", "masked-marginals", "pseudo-ppl")]
CASES += [("msa_t2_tiny", "masked-marginals")]


def score(fixture, name, strategy, tmp_path, model):
    from esm_b200 import Alphabet, predict_cli
    alphabet = Alphabet.from_architecture("msa_transformer" if name.startswith("msa") else "ESM-1b")
    return predict_cli.score_model(model, alphabet, name.startswith("msa"), cli_args(fixture, strategy, tmp_path),
                                   mutations(fixture))


# ---- the kernel -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", [33, 35])
@pytest.mark.parametrize("n", [1, 1000, 100000])
def test_log_softmax_rows_matches_torch(V, n):
    from esm_b200.variants import log_softmax_rows
    g = torch.Generator(device="cuda").manual_seed(n + V)
    buf = (torch.rand((n, 64), device="cuda", generator=g) * 160 - 80)  # ld = 64, logits in [-80, 80]
    logits = buf[:, :V]
    want = torch.log_softmax(logits, dim=-1)
    got = log_softmax_rows(logits)
    assert got.shape == (n, V)
    assert float((got - want).abs().max()) <= 2e-6
    target = torch.randint(0, V, (n,), device="cuda", generator=g)
    got_t = log_softmax_rows(logits, target)
    assert float((got_t - want.gather(1, target[:, None])[:, 0]).abs().max()) <= 2e-6
    with pytest.raises(ValueError):
        log_softmax_rows(logits, torch.full((n,), V, device="cuda"))


def test_log_softmax_rows_argument_checks():
    from esm_b200 import _lib
    lib = _lib.load()
    x = torch.zeros((4, 128), device="cuda")
    out = torch.empty((4, 128), device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    assert lib.esmb200_log_softmax_rows(x.data_ptr(), 128, 4, 65, None, out.data_ptr(), s) == -1  # V > 64
    assert lib.esmb200_log_softmax_rows(x.data_ptr(), 32, 4, 33, None, out.data_ptr(), s) == -1   # ld < V
    assert lib.esmb200_log_softmax_rows(None, 64, 4, 33, None, out.data_ptr(), s) == -1
    assert lib.esmb200_log_softmax_rows(x.data_ptr(), 64, 0, 33, None, out.data_ptr(), s) == 0


# ---- predict.py's outputs ---------------------------------------------------------------------------------------
def _compare(got, want, centered=False):
    """(rel-Fro, max-abs / rms of the reference) of two score vectors; centered: both minus their mean first."""
    got, want = torch.tensor(got, dtype=torch.float64), torch.tensor(want, dtype=torch.float64)
    if centered:
        got, want = got - got.mean(), want - want.mean()
    rms = float(want.pow(2).mean().sqrt())
    return float((got - want).norm() / want.norm()), float((got - want).abs().max()) / rms, rms


# Pseudo-ppl scores share a large common offset (a sum of ~50 log-probabilities, about -1000 here) while mutants differ
# by a few tens, so the uncentered comparison alone would let an error of the size of the whole between-mutant signal
# pass. Each pseudo-ppl is therefore also compared centered (minus the mean over the mutants). The fp16 bound there is
# wider than the logits tolerance because the sum adds up the errors of ~50 independent fp16 log-probabilities while
# the centered signal is a single-residue effect; an indexing or summation slip moves a score by tens and still fails
# it, and the fp32x3 test below holds the centered comparison to the logits tolerance.
PPPL_CENTERED_FP16 = 2e-2


@pytest.mark.parametrize("name,strategy", CASES)
def test_scores_match_predict_py(fixture, name, strategy, tmp_path):
    _, want = reference_table(fixture, name, strategy)
    got = score(fixture, name, strategy, tmp_path, fixture_model(fixture, name))
    r, m, rms = _compare(got, want)
    assert rms >= 0.05, "the fixture's scores are flat: the comparison would be vacuous"
    line = f"PARITY variants {name} {strategy}: rel_fro={r:.3e} max_abs/rms={m:.3e} (rms {rms:.3g})"
    ok = r <= REL_FRO and m <= MAX_ABS_RMS
    if strategy == "pseudo-ppl":
        rc, mc, rmsc = _compare(got, want, centered=True)
        assert rmsc >= 0.05, "the fixture's pseudo-ppl scores do not vary between mutants"
        line += f"; centered rel_fro={rc:.3e} max_abs/rms={mc:.3e} (rms {rmsc:.3g})"
        ok = ok and rc <= PPPL_CENTERED_FP16 and mc <= 2.5 * PPPL_CENTERED_FP16
    print(line)
    assert ok


@pytest.mark.parametrize("name,strategy", [c for c in CASES if not c[0].startswith("msa")])
def test_fp32x3_scores_are_10x_closer(fixture, name, strategy, tmp_path):
    _, want = reference_table(fixture, name, strategy)
    centered = strategy == "pseudo-ppl"
    r16 = _compare(score(fixture, name, strategy, tmp_path, fixture_model(fixture, name)), want, centered)[0]
    got32 = score(fixture, name, strategy, tmp_path, fixture_model(fixture, name, "fp32x3"))
    r32, m32, _ = _compare(got32, want, centered)
    print(f"PARITY variants fp32x3 {name} {strategy}{' centered' if centered else ''}: rel_fro={r32:.3e} "
          f"max_abs/rms={m32:.3e} (fp16 {r16:.3e})")
    assert r32 * 10 <= r16
    assert r32 <= REL_FRO and m32 <= MAX_ABS_RMS


def test_half_model_scores(fixture, tmp_path):
    """model.half(): fp16-rounded weights, fp32 log-probabilities, within the tolerance of the fp32 model's scores."""
    from esm_b200 import variants
    for name in ("esm2_t2_tiny", "esm1b_t2_tiny"):
        model = fixture_model(fixture, name)
        want = score(fixture, name, "masked-marginals", tmp_path, model)
        model = model.half()
        _, _, tokens = model.alphabet.get_batch_converter()([("p", fixture["sequence"])])
        assert variants.masked_marginals(model, tokens).dtype == torch.float32
        got = score(fixture, name, "masked-marginals", tmp_path, model)
        rms = math.sqrt(sum(v * v for v in want) / len(want))
        r = rel_fro(got, want)
        m = float((torch.tensor(got) - torch.tensor(want)).abs().max())
        print(f"PARITY variants half() {name}: rel_fro={r:.3e} max_abs/rms={m / rms:.3e} vs the fp32 model")
        assert r <= REL_FRO and m <= MAX_ABS_RMS * rms


# ---- batching is exact ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["esm2_t2_tiny", "esm1b_t2_tiny", "msa_t2_tiny"])
def test_masked_marginals_do_not_depend_on_the_chunk_size(fixture, name, tmp_path):
    from esm_b200 import variants
    model = fixture_model(fixture, name)
    if name.startswith("msa"):
        data = [variants.read_msa(cli_args(fixture, "masked-marginals", tmp_path).msa_path, fixture["msa_samples"])]
    else:
        data = [("p", fixture["sequence"])]
    _, _, tokens = model.alphabet.get_batch_converter()(data)
    per_copy = tokens[0].numel()
    full = variants.masked_marginals(model, tokens, max_tokens=1 << 30)
    assert full.shape == (tokens.shape[-1], model.alphabet_size)
    for copies in (1, 7):
        assert torch.equal(variants.masked_marginals(model, tokens, max_tokens=copies * per_copy), full), copies
    assert torch.equal(variants.masked_marginals(model, tokens, max_tokens=1), full)  # at least one copy per chunk
    sub = variants.masked_marginals(model, tokens, positions=[5, 2, 9])
    assert torch.equal(sub, full[[5, 2, 9]])
    # the row-gathered head equals the full head of model(...)["logits"], through the same kernel
    tokens = tokens.cuda()
    for i in range(tokens.shape[-1]):
        masked = tokens.clone()
        if tokens.dim() == 3:
            masked[0, 0, i] = model.mask_idx
            row = model(masked)["logits"][0, 0, i:i + 1]
        else:
            masked[0, i] = model.mask_idx
            row = model(masked)["logits"][0, i:i + 1]
        assert torch.equal(variants.log_softmax_rows(row.contiguous()), full[i:i + 1]), i


def test_pseudo_ppl_batched_across_mutants_equals_one_at_a_time(fixture):
    from esm_b200 import variants
    model = fixture_model(fixture, "esm2_t2_tiny")
    muts = mutations(fixture)[:9]
    seq, off = fixture["sequence"], fixture["offset_idx"]
    batched = variants.pseudo_ppl(model, model.alphabet, seq, muts, off)
    single = [variants.pseudo_ppl(model, model.alphabet, seq, [m], off, max_tokens=1)[0] for m in muts]
    assert batched == single
    chunked = variants.pseudo_ppl(model, model.alphabet, seq, muts, off, max_tokens=13 * (len(seq) + 2))
    assert batched == chunked


# ---- full size against the reference, predict.py's batch-1 loop, eager fp32 on the same GPU ------------------------
def _centered_rel_fro(got, want):
    got = got.double() - got.double().mean(-1, keepdim=True)
    want = want.double() - want.double().mean(-1, keepdim=True)
    return float((got - want).norm() / want.norm())


def test_esm1v_650M_masked_marginals_against_the_reference(esm_ref):
    from esm_b200 import ProteinBertModel, variants
    from esm1b_weights import make_esm1b_state_dict
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    L, E, H = 33, 1280, 20
    args = argparse.Namespace(arch="roberta_large", layers=L, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                              max_positions=1024, emb_layer_norm_before=True, token_dropout=True)
    sd = make_esm1b_state_dict(L, E, H, seed=0)
    alphabet = esm_ref.Alphabet.from_architecture("roberta_large")
    _, _, tokens = alphabet.get_batch_converter()([("protein1", BLAT_ECOLX)])
    ref = esm_ref.ProteinBertModel(args, alphabet)
    ref.load_state_dict(sd, strict=True)
    ref = ref.eval().cuda()
    rows = []
    with torch.no_grad():
        for i in range(tokens.size(1)):  # predict.py:206-214
            masked = tokens.clone()
            masked[0, i] = alphabet.mask_idx
            rows.append(torch.log_softmax(ref(masked.cuda())["logits"], dim=-1)[:, i])
    want = torch.cat(rows)
    del ref
    torch.cuda.empty_cache()
    model = ProteinBertModel(args, "roberta_large")
    model.load_state_dict(sd, strict=True)
    got = variants.masked_marginals(model.eval().cuda(), tokens)
    r = _centered_rel_fro(got, want)
    print(f"PARITY variants reference_eager_esm1v_650M BLAT_ECOLX masked-marginals T={tokens.size(1)}: "
          f"centered rel_fro={r:.3e}", flush=True)
    assert got.shape == want.shape == (265, 33)
    assert r <= REL_FRO


def test_msa_transformer_masked_marginals_against_the_reference(esm_ref):
    from esm_b200 import MSATransformer, variants
    from oracle.msa_oracle import make_msa_state_dict, make_msa_tokens
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    L, E, Fd, H = 12, 768, 3072, 12
    args = argparse.Namespace(layers=L, embed_dim=E, ffn_embed_dim=Fd, attention_heads=H, dropout=0.0,
                              attention_dropout=0.0, activation_dropout=0.0, max_tokens_per_msa=2 ** 14,
                              max_tokens=2 ** 14, max_positions=1024, embed_positions_msa=True)
    sd = make_msa_state_dict(L, E, Fd, H, seed=0)
    tokens = make_msa_tokens(1, 64, 101, seed=7)  # unpadded 64 x 100 alignment (+ <cls>)
    positions = list(range(0, 101, 7))[:16]
    ref = esm_ref.MSATransformer(args, esm_ref.Alphabet.from_architecture("msa_transformer"))
    ref.load_state_dict(sd, strict=True)
    ref = ref.eval().cuda()
    mask_idx = ref.mask_idx
    rows = []
    with torch.no_grad():
        for i in positions:  # predict.py:170-177
            masked = tokens.clone()
            masked[0, 0, i] = mask_idx
            rows.append(torch.log_softmax(ref(masked.cuda())["logits"], dim=-1)[:, 0, i])
        ref_logits = ref(tokens.cuda())["logits"][0, 0].float().cpu()
    want = torch.cat(rows)
    del ref
    torch.cuda.empty_cache()
    model = MSATransformer(args, "msa_transformer")
    model.load_state_dict(sd, strict=True)
    model = model.eval().cuda()
    got = variants.masked_marginals(model, tokens, positions=positions)  # one chunk of 16 copies
    # At this size too, the scorer equals MSATransformer.forward on each masked copy, one at a time, put through the
    # same kernel, bit for bit: batching 16 copies and reading one row per copy adds nothing.
    tok = tokens.cuda()
    for k, i in enumerate(positions):
        masked = tok.clone()
        masked[0, 0, i] = model.mask_idx
        row = model(masked)["logits"][0, 0, i:i + 1].contiguous()
        assert torch.equal(variants.log_softmax_rows(row), got[k:k + 1]), i
    # The library's own forward of the unmasked alignment against the reference's, for the size of the stack's error.
    with torch.no_grad():
        fwd = model(tok)["logits"][0, 0].float().cpu()
    r = _centered_rel_fro(got, want)
    rf = _centered_rel_fro(fwd, ref_logits)
    print(f"PARITY variants reference_eager_msa_transformer 64x100 masked-marginals 16 columns: "
          f"centered rel_fro={r:.3e}; forward logits of row 0 without a mask: centered rel_fro={rf:.3e}", flush=True)
    # Since the scorer is the forward bit for bit, the remaining difference is the fp16-mode error of the 12-layer axial
    # stack with 64 tied rows on these random weights (measured at 1.0e-2 on an H100), which the unmasked forward shows
    # as well (test_masked_marginals_fp32x3_against_the_reference in test_gpu_msa_precision.py runs the same comparison
    # in the fp32x3 mode). Held to that level, not to the 4e-3 of the sequence models.
    assert r <= 2e-2 and rf <= 2e-2


# ---- the command line -----------------------------------------------------------------------------------------------
def test_cli_end_to_end_matches_predict_py(fixture, tmp_path):
    import variant_fixtures as vf
    from esm_b200 import predict_cli
    (tmp_path / "dms.csv").write_text(fixture["dms_csv"])
    (tmp_path / "msa.a3m").write_text(fixture["a3m"])
    names = ["esm2_t2_tiny", "esm1b_t2_tiny", "msa_t2_tiny"]
    paths = [vf.write_checkpoint(n, vf.MODELS[n], str(tmp_path)) for n in names]
    out = tmp_path / "out.csv"
    args = predict_cli.create_parser().parse_args(
        ["--model-location"] + paths + ["--sequence", fixture["sequence"], "--dms-input", str(tmp_path / "dms.csv"),
                                        "--dms-output", str(out), "--offset-idx", str(fixture["offset_idx"]),
                                        "--scoring-strategy", "masked-marginals", "--msa-path",
                                        str(tmp_path / "msa.a3m"), "--msa-samples", str(fixture["msa_samples"])])
    predict_cli.run(args)
    got = list(csv.reader(io.StringIO(out.read_text())))
    first, _ = reference_table(fixture, names[0], "masked-marginals")
    assert got[0] == first[0][:-1] + paths
    assert [r[:4] for r in got] == [r[:4] for r in first]  # index and input columns, strings exact
    for j, n in enumerate(names):
        _, want = reference_table(fixture, n, "masked-marginals")
        col = [float(r[4 + j]) for r in got[1:]]
        rms = math.sqrt(sum(v * v for v in want) / len(want))
        assert rel_fro(col, want) <= REL_FRO
        assert max(abs(a - b) for a, b in zip(col, want)) <= MAX_ABS_RMS * rms
