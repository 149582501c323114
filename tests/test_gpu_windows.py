"""GPU (-m gpu): overlapping windows for long proteins (esm_b200.windows, ProteinLanguageModel.forward_windowed, the
windowed variant scorers and the --window flag of both command lines).

  * esmb200_window_merge against a float64 restatement, past its launch's grid cap, into a poisoned output wider
    than C; bit-reproducible; one-term rows copied bit for bit;
  * proteins within the window: forward_windowed and the three scorers bit-identical to the unwindowed path;
  * longer proteins (an ESM-1b-shaped model with 64 learned positions, and ESM-2): every merged row against a float64
    merge of what forward gives on each window alone; bit-identical for any max_tokens;
  * the unmodified reference run on each window crop (tests/golden/windows/*.pt, made by
    tests/golden/make_golden_windows.py), merged with the documented weights, at the ESM-1b golden tolerances;
  * predict_cli --window and extract_cli --window end to end.
"""
import argparse
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # esm1b_weights

pytestmark = pytest.mark.gpu

REL_FRO = 3e-3          # DESIGN.md section 4, as tests/test_gpu_esm1b.py holds the ESM-1b golden files
REL_FRO_LOGITS = 4e-3
U = 2.0 ** -24
GOLDEN = os.path.join("windows", "esm1b_L2_E128_H2_P64")


def rel_fro(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def centered_rel_fro(got, want):
    got = got.double() - got.double().mean(-1, keepdim=True)
    want = want.double() - want.double().mean(-1, keepdim=True)
    return float((got - want).norm() / want.norm())


def checksum(sd):
    return float(sum(v.double().abs().sum() for k, v in sorted(sd.items())))


def esm1b_model(max_positions=64, L=2, E=128, H=2):
    from esm_b200 import ProteinBertModel
    from esm1b_weights import make_esm1b_state_dict
    args = argparse.Namespace(arch="roberta_large", layers=L, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                              max_positions=max_positions, emb_layer_norm_before=True, token_dropout=True)
    model = ProteinBertModel(args, "ESM-1b")
    model.load_state_dict(make_esm1b_state_dict(L, E, H, seed=0, max_positions=max_positions), strict=True)
    return model.eval().cuda()


def esm2_model(L=2, E=128, H=2):
    from esm_b200 import ESM2
    from oracle.weights import make_state_dict
    model = ESM2(num_layers=L, embed_dim=E, attention_heads=H)
    model.load_state_dict(make_state_dict(L, E, H, seed=0), strict=True)
    return model.eval().cuda()


def protein(n, seed):
    g = torch.Generator().manual_seed(seed)
    return "".join("LAGVSERTIDPKQNFYMHWC"[i] for i in torch.randint(0, 20, (n,), generator=g).tolist())


# ---- the kernel -------------------------------------------------------------------------------------------------
def merge_f64(src, idx, w, seg):
    """The float64 merge and the sum of its terms' magnitudes, [rows, C] each: every term w[j] * src[idx[j]] added into
    its row r (seg[r] <= j < seg[r + 1]) by index_add_."""
    s, i, ww, sg = src.double().cpu(), idx.cpu(), w.double().cpu(), seg.cpu()
    rows = sg.numel() - 1
    row_of = torch.repeat_interleave(torch.arange(rows), sg.diff())
    terms = ww[:, None] * s[i]
    out = torch.zeros((rows, s.shape[1]), dtype=torch.float64).index_add_(0, row_of, terms)
    mag = torch.zeros_like(out).index_add_(0, row_of, terms.abs_())
    return out, mag


POISON = 0x7FA5A5A5  # a NaN no fp32 operation produces: it marks output elements the kernel must not touch or skipped


# 5120 x 3500: 17.9 M elements, past the launch's 65,536 blocks of 256 threads, so the grid-stride loop runs (a 15B
# representation merged over a protein of about 3,300 residues)
@pytest.mark.parametrize("C,rows", [(1, 400), (33, 400), (64, 400), (1280, 120), (5120, 3500)])
def test_merge_matches_float64_and_copies_single_terms(C, rows):
    from esm_b200 import _lib, windows
    g = torch.Generator().manual_seed(C)
    R = 3 * rows
    ld = C + 7                                                                 # a row stride wider than C
    buf = torch.randn((R, ld), generator=g) * 10
    counts = torch.randint(1, 6, (rows,), generator=g)
    seg = torch.zeros(rows + 1, dtype=torch.int64)
    seg[1:] = counts.cumsum(0)
    idx = torch.randint(0, R, (int(seg[-1]),), generator=g)
    w = torch.rand((int(seg[-1]),), generator=g) + 0.05
    # special values in the source rows of one-term segments: copied bit for bit whatever the weight
    single = torch.nonzero(counts == 1)[:, 0]
    srows = idx[seg[single]]
    buf[srows, 0] = -0.0
    if C > 1:
        buf[srows[: len(srows) // 2], 1] = float("nan")
        buf[srows[len(srows) // 2:], C - 1] = float("-inf")
    src = buf.cuda()[:, :C]
    assert src.stride(0) == ld
    got = windows.merge_rows(src, idx, w, seg)
    again = windows.merge_rows(src, idx, w, seg)
    assert got.shape == (rows, C)
    assert torch.equal(got.view(torch.int32), again.view(torch.int32))        # bit-reproducible
    # through the C ABI into a poisoned output 5 columns wider than C: every element written, no padding column touched
    out_ld = C + 5
    poisoned = torch.full((rows, out_ld), POISON, dtype=torch.int32, device="cuda").view(torch.float32)
    dev = lambda t, dt: t.to("cuda", dt).contiguous()  # noqa: E731
    idx_d, w_d, seg_d = dev(idx, torch.int64), dev(w, torch.float32), dev(seg, torch.int64)
    _lib.check(_lib.load().esmb200_window_merge(src.data_ptr(), ld, idx_d.data_ptr(), w_d.data_ptr(), seg_d.data_ptr(),
                                                rows, C, poisoned.data_ptr(), out_ld,
                                                torch.cuda.current_stream().cuda_stream))
    bits = poisoned.view(torch.int32)
    assert bool((bits[:, C:] == POISON).all()), "a padding column was written"
    assert torch.equal(bits[:, :C], got.view(torch.int32)), "an element was not written, or differs between calls"
    s = src.cpu()
    copied = got.cpu()[single]
    assert torch.equal(copied.view(torch.int32), s[srows].contiguous().view(torch.int32))
    multi = counts > 1
    want, mag = merge_f64(s, idx, w, seg)
    g64 = got.cpu().double()[multi]
    want, mag = want[multi], mag[multi]
    fin = torch.isfinite(want)                      # the special values also feed some multi-term rows
    assert torch.equal(g64.isnan(), want.isnan()) and torch.equal(g64[want.isinf()], want[want.isinf()])
    err = (g64 - want)[fin].abs()
    bound = 6 * U * mag[fin] + 1e-30
    assert bool((err <= bound).all()), float((err / bound).max())
    print(f"PARITY window_merge C={C} rows={rows} ({rows * C / 1e6:.2f} M elements): max err/bound "
          f"{float((err / bound).max()):.3f} (bound 6u sum|w x|); poisoned output with out_ld = C + 5: every element "
          f"written, no padding column touched")


def test_merge_argument_checks():
    from esm_b200 import _lib
    lib = _lib.load()
    x = torch.zeros((4, 64), device="cuda")
    out = torch.empty((4, 64), device="cuda")
    idx = torch.zeros(4, dtype=torch.int64, device="cuda")
    w = torch.ones(4, device="cuda")
    seg = torch.arange(5, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()
    assert lib.esmb200_window_merge(p(x), 64, p(idx), p(w), p(seg), 4, 0, p(out), 64, s) == -1    # C == 0
    assert lib.esmb200_window_merge(p(x), 32, p(idx), p(w), p(seg), 4, 33, p(out), 64, s) == -1   # src_ld < C
    assert lib.esmb200_window_merge(p(x), 64, p(idx), p(w), p(seg), 4, 33, p(out), 16, s) == -1   # out_ld < C
    assert lib.esmb200_window_merge(p(x), 64, p(idx), p(w), p(seg), -1, 33, p(out), 64, s) == -1  # rows < 0
    assert lib.esmb200_window_merge(None, 64, p(idx), p(w), p(seg), 4, 33, p(out), 64, s) == -1
    assert lib.esmb200_window_merge(None, 64, None, None, None, 0, 33, None, 64, s) == 0           # nothing to do
    assert lib.esmb200_window_merge(p(x), 64, p(idx), p(w), p(seg), 4, 64, p(out), 64, s) == 0
    torch.cuda.synchronize()


# ---- proteins within the window: the unwindowed path, bit for bit ------------------------------------------------
def _golden_model(golden_dir, name):
    from esm1b_weights import make_esm1b_state_dict
    from esm_b200 import ESM2, ProteinBertModel
    from oracle.weights import make_state_dict
    fx = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    c = fx["config"]
    if "model_args" in c:
        args = c["model_args"]
        model = ProteinBertModel(argparse.Namespace(**args), "ESM-1b")
        sd = make_esm1b_state_dict(c["num_layers"], c["embed_dim"], c["attention_heads"], seed=c["seed"],
                                   emb_layer_norm_before=args["emb_layer_norm_before"])
    else:
        model = ESM2(num_layers=c["num_layers"], embed_dim=c["embed_dim"], attention_heads=c["attention_heads"])
        sd = make_state_dict(c["num_layers"], c["embed_dim"], c["attention_heads"], seed=c["seed"])
    model.load_state_dict(sd, strict=True)
    return model.eval().cuda(), fx["tokens"]


@pytest.mark.parametrize("name", ["tiny_L2_E128_H2", "nopad_L2_E128_H2", "esm1b_tiny_L2_E128_H2",
                                  "esm1b_mid_L3_E256_H4"])
def test_forward_windowed_within_the_window_is_forward(golden_dir, name):
    model, tokens = _golden_model(golden_dir, name)
    tokens = tokens.cuda()
    N = model.num_layers
    layers = [0, 1, N]
    want = model(tokens, repr_layers=layers)
    keep = tokens.ne(model.padding_idx)
    for W in (tokens.shape[1] - 2, tokens.shape[1] + 100):
        for max_tokens in (None, 1):
            got = model.forward_windowed(tokens, W, repr_layers=layers, max_tokens=max_tokens)
            for key, a, b in [("logits", got["logits"], want["logits"])] + [
                    (f"repr {i}", got["representations"][i], want["representations"][i]) for i in layers]:
                for r in range(tokens.shape[0]):
                    n = int(keep[r].nonzero().max()) + 1
                    assert torch.equal(a[r, :n].view(torch.int32), b[r, :n].view(torch.int32)), (key, r)
                    assert not bool(a[r, n:].any()), (key, r)                    # pad rows are zero
    print(f"PARITY windows {name}: forward_windowed within the window bit-identical to forward")


@pytest.mark.parametrize("kind", ["esm2", "esm1b"])
def test_scorers_within_the_window_are_unchanged(kind):
    from esm_b200 import variants
    model = esm2_model() if kind == "esm2" else esm1b_model(max_positions=1024)
    seq = protein(60, 7)
    muts = [f"{seq[i]}{i}{'A' if seq[i] != 'A' else 'C'}" for i in (0, 11, 30, 59)]
    _, _, tokens = model.alphabet.get_batch_converter()([("p", seq)])
    for W in (60, 1000):
        assert torch.equal(variants.masked_marginals(model, tokens, window=W), variants.masked_marginals(model, tokens))
        assert torch.equal(variants.masked_marginals(model, tokens, positions=[3, 0, 61], max_tokens=62, window=W),
                           variants.masked_marginals(model, tokens, positions=[3, 0, 61], max_tokens=62))
        assert torch.equal(variants.wt_marginals(model, tokens, window=W), variants.wt_marginals(model, tokens))
        assert (variants.pseudo_ppl(model, model.alphabet, seq, muts, window=W)
                == variants.pseudo_ppl(model, model.alphabet, seq, muts))


# ---- longer proteins: a float64 merge of each window run alone --------------------------------------------------
def _windows_alone(model, tokens_row, W):
    """Each window's tokens (tokenised as a protein of its own, no padding) and forward on it alone."""
    from esm_b200 import windows
    T = tokens_row.numel()
    plan = windows.Plan(T - 2, W, 1, 1)
    ext = torch.cat([tokens_row.cpu(), torch.tensor([model.padding_idx])])
    wt = ext[plan.gather(T, plan.tokens)]
    return plan, wt


def _merge_terms_f64(plan, per_window, T):
    """float64 merge of per_window[k] [Tw, C] tensors with the documented weights, recomputed here."""
    W, S, K = plan.W, plan.starts, plan.K
    C = per_window[0].shape[-1]
    out = torch.zeros((T, C), dtype=torch.float64)
    mag = torch.zeros_like(out)
    out[0] = per_window[0][0].double()
    out[T - 1] = per_window[K - 1][plan.width + 1].double()
    for p in range(T - 2):
        cover = [(k, p - s) for k, s in enumerate(S) if s <= p < s + plan.width]
        taper = [min(o + 1, W - o) for _, o in cover]
        for (k, o), t in zip(cover, taper):
            v = (t / sum(taper)) * per_window[k][1 + o].double()
            out[1 + p] += v
            mag[1 + p] += v.abs()
    return out, mag


@pytest.mark.parametrize("kind", ["esm1b", "esm2"])
def test_forward_windowed_long_proteins_match_a_float64_merge(kind):
    model = esm1b_model() if kind == "esm1b" else esm2_model()
    W = 62
    lengths = [150, 40, 101]
    seqs = [protein(n, 11 + n) for n in lengths]
    _, _, tokens = model.alphabet.get_batch_converter()([(str(i), s) for i, s in enumerate(seqs)])
    tokens = tokens.cuda()
    N = model.num_layers
    got = model.forward_windowed(tokens, W, repr_layers=[0, 1, N])
    for max_tokens in (1, 5 * (W + 2), 10 ** 7):
        again = model.forward_windowed(tokens, W, repr_layers=[0, 1, N], max_tokens=max_tokens)
        assert torch.equal(again["logits"], got["logits"]), max_tokens
        for i in (0, 1, N):
            assert torch.equal(again["representations"][i], got["representations"][i]), (max_tokens, i)
    worst = 0.0
    for b, n in enumerate(lengths):
        T = n + 2
        plan, wt = _windows_alone(model, tokens[b, :T], W)
        outs = [model(wt[k:k + 1].cuda(), repr_layers=[0, 1, N]) for k in range(plan.K)]
        for key, get in [("logits", lambda o: o["logits"][0])] + [
                (f"repr {i}", (lambda i: lambda o: o["representations"][i][0])(i)) for i in (0, 1, N)]:
            want, mag = _merge_terms_f64(plan, [get(o).cpu() for o in outs], T)
            g = (got["logits"] if key == "logits" else got["representations"][int(key.split()[1])])[b]
            err = (g[:T].cpu().double() - want).abs()
            bound = 4 * U * mag + 1e-30
            worst = max(worst, float((err / bound).max()))
            assert bool((err <= bound).all()), (b, key, float((err / bound).max()))
            assert not bool(g[T:].any())
    print(f"PARITY windows {kind} W={W} lengths {lengths}: merged rows within {worst:.3f} of 4u sum|w x| of a float64 "
          f"merge of the windows run alone; bit-identical for max_tokens 1, 5 windows, all")


@pytest.mark.parametrize("kind", ["esm1b", "esm2"])
def test_scorers_long_proteins_match_a_float64_merge(kind):
    from esm_b200 import variants
    model = esm1b_model() if kind == "esm1b" else esm2_model()
    W = 62
    seq = protein(150, 5)
    _, _, tokens = model.alphabet.get_batch_converter()([("p", seq)])
    T = tokens.shape[1]
    plan, wt = _windows_alone(model, tokens[0], W)
    mask = model.mask_idx

    def merged_masked_logits(tok_row, t):
        """float64 merge of the masked position t's logits in each covering window's masked copy."""
        plan_, wt_ = _windows_alone(model, tok_row, W)
        rows, taper = [], []
        if t == 0:
            cover = [(0, 0, 1)]
        elif t == T - 1:
            cover = [(plan_.K - 1, plan_.width + 1, 1)]
        else:
            cover = [(k, t - s, min(t - s, W - t + s + 1)) for k, s in enumerate(plan_.starts) if s <= t - 1 < s + W]
        copies = []
        for k, r, _ in cover:
            c = wt_[k].clone()
            c[r] = mask
            copies.append(c)
        logits = model(torch.stack(copies).cuda())["logits"].cpu().double()
        tot = sum(tp for _, _, tp in cover)
        return sum((tp / tot) * logits[j, r] for j, (_, r, tp) in enumerate(cover))

    positions = [0, 1, 2, 30, 45, 60, 89, 100, 148, 150, 151]
    got = variants.masked_marginals(model, tokens, positions=positions, window=W)
    want = torch.stack([torch.log_softmax(merged_masked_logits(tokens[0], t), -1) for t in positions])
    assert float((got.cpu().double() - want).abs().max()) <= 1e-5
    full = variants.masked_marginals(model, tokens, window=W)
    for max_tokens in (1, 7 * (W + 2)):
        assert torch.equal(variants.masked_marginals(model, tokens, max_tokens=max_tokens, window=W), full)
    assert torch.equal(full[positions], got)
    # wt-marginals: log_softmax of the merged logits of the windows run alone
    outs = [model(wt[k:k + 1].cuda())["logits"][0].cpu() for k in range(plan.K)]
    want_wt = torch.log_softmax(_merge_terms_f64(plan, outs, T)[0], -1)
    got_wt = variants.wt_marginals(model, tokens, window=W)
    assert float((got_wt.cpu().double() - want_wt).abs().max()) <= 1e-5
    # pseudo-ppl: compute_pppl's indexing on the full mutated sequence, each masked position merged over its windows
    muts = [f"{seq[i]}{i}{'W' if seq[i] != 'W' else 'C'}" for i in (3, 77)]
    got_pp = variants.pseudo_ppl(model, model.alphabet, seq, muts, window=W)
    assert got_pp == variants.pseudo_ppl(model, model.alphabet, seq, muts, max_tokens=1, window=W)
    for m, score in zip(muts, got_pp):
        idx = int(m[1:-1])
        s = seq[:idx] + m[-1] + seq[idx + 1:]
        _, _, tok = model.alphabet.get_batch_converter()([("m", s)])
        want_pp = 0.0
        for i in range(1, len(s) - 1):
            lp = torch.log_softmax(merged_masked_logits(tok[0], i), -1)
            want_pp += float(lp[model.alphabet.get_idx(s[i])])
        assert abs(score - want_pp) <= 1e-3, (m, score, want_pp)
    print(f"PARITY windows {kind} scorers W={W} n=150: masked/wt within 1e-5 of a float64 merge, pseudo-ppl within "
          f"1e-3; bit-identical for every max_tokens")


# ---- the reference on each window crop ---------------------------------------------------------------------------
def test_matches_the_reference_on_window_crops(golden_dir):
    from esm_b200 import variants, windows
    from esm1b_weights import make_esm1b_state_dict
    fx = torch.load(os.path.join(golden_dir, GOLDEN + ".pt"), weights_only=False)
    c = fx["config"]
    args = c["model_args"]
    sd = make_esm1b_state_dict(c["num_layers"], c["embed_dim"], c["attention_heads"], seed=c["seed"],
                               emb_layer_norm_before=True, max_positions=args["max_positions"])
    assert abs(checksum(sd) - fx["state_dict_checksum"]) <= 1e-6 * fx["state_dict_checksum"]
    model = esm1b_model(max_positions=args["max_positions"], L=c["num_layers"], E=c["embed_dim"],
                        H=c["attention_heads"])
    W, seq, L = fx["window"], fx["sequence"], c["num_layers"]
    plan = windows.Plan(len(seq), W, 1, 1)
    assert plan.starts == fx["starts"]
    _, _, tokens = model.alphabet.get_batch_converter()([("p", seq)])
    T = tokens.shape[1]
    assert T > args["max_positions"]
    ext = torch.cat([tokens[0], torch.tensor([model.padding_idx])])
    assert torch.equal(ext[plan.gather(T, W + 2)], fx["window_tokens"])
    with pytest.raises(ValueError):
        model(tokens.cuda())                                                  # too long without a window
    got = model.forward_windowed(tokens.cuda(), W, repr_layers=[L])
    want_logits = _merge_terms_f64(plan, list(fx["logits"]), T)[0]
    want_repr = _merge_terms_f64(plan, list(fx["representations"]), T)[0]
    rl = rel_fro(got["logits"][0].cpu(), want_logits)
    rr = rel_fro(got["representations"][L][0].cpu(), want_repr)
    positions = sorted(fx["masked"])
    lp = variants.masked_marginals(model, tokens, positions=positions, window=W).cpu()
    want_lp = []
    for t in positions:
        cover = fx["masked"][t]
        if t == 0 or t == T - 1:
            wts = [1.0]
        else:
            taper = [min(r, W - r + 1) for _, r, _ in cover]  # offset o = r - 1
            wts = [x / sum(taper) for x in taper]
        assert [k for k, _, _ in cover] == sorted(k for k, s in enumerate(plan.starts)
                                                    if (t == 0 and k == 0) or (t == T - 1 and k == plan.K - 1)
                                                    or (0 < t < T - 1 and s <= t - 1 < s + W))
        want_lp.append(torch.log_softmax(sum(w * row.double() for w, (_, _, row) in zip(wts, cover)), -1))
    rm = centered_rel_fro(lp, torch.stack(want_lp))
    print(f"PARITY windows reference {GOLDEN}: logits rel_fro={rl:.3e} repr rel_fro={rr:.3e} masked-marginals "
          f"centered rel_fro={rm:.3e}")
    assert rl <= REL_FRO_LOGITS and rr <= REL_FRO and rm <= REL_FRO_LOGITS


# ---- the command lines ---------------------------------------------------------------------------------------------
def _checkpoint(tmp_path, max_positions=64):
    """An ESM-1b checkpoint with 64 learned positions, in the v1 format the loaders read."""
    from esm1b_weights import make_esm1b_state_dict
    sd = make_esm1b_state_dict(2, 128, 2, seed=0, max_positions=max_positions)
    reg = ("contact_head.regression.weight", "contact_head.regression.bias")
    args = argparse.Namespace(arch="roberta_large", layers=2, embed_dim=128, ffn_embed_dim=512, attention_heads=2,
                              max_positions=max_positions, emb_layer_norm_before=True, token_dropout=True)
    path = str(tmp_path / "esm1b_t2_window.pt")
    torch.save({"args": args, "model": {k: v for k, v in sd.items() if k not in reg}}, path)
    torch.save({"model": {k: sd[k] for k in reg}}, str(tmp_path / "esm1b_t2_window-contact-regression.pt"))
    return path


@pytest.mark.parametrize("strategy", ["masked-marginals", "wt-marginals", "pseudo-ppl"])
def test_predict_cli_window(tmp_path, strategy):
    import csv
    from esm_b200 import predict_cli, variants
    path = _checkpoint(tmp_path)
    seq = protein(150, 5)
    muts = [f"{seq[i]}{i}{'W' if seq[i] != 'W' else 'C'}" for i in (0, 30, 75, 149)]
    (tmp_path / "dms.csv").write_text("mutant,score\n" + "".join(f"{m},0.5\n" for m in muts))
    out = tmp_path / "out.csv"
    args = predict_cli.create_parser().parse_args(
        ["--model-location", path, "--sequence", seq, "--dms-input", str(tmp_path / "dms.csv"), "--dms-output",
         str(out), "--scoring-strategy", strategy, "--window", "62"])
    predict_cli.run(args)
    col = [float(r[-1]) for r in list(csv.reader(out.open()))[1:]]
    model, alphabet, _ = predict_cli.load_model(path)
    model = model.eval().cuda()
    _, _, tokens = alphabet.get_batch_converter()([("protein1", seq)])
    if strategy == "pseudo-ppl":
        want = variants.pseudo_ppl(model, alphabet, seq, muts, window=62)
    else:
        lp = (variants.masked_marginals(model, tokens, window=62) if strategy == "masked-marginals"
              else variants.wt_marginals(model, tokens, window=62))
        want = variants.label_scores(lp, alphabet, seq, muts)
    assert col == want
    args.window = None
    with pytest.raises(ValueError):
        predict_cli.run(args)                                                 # 152 tokens > 64 positions


def test_extract_cli_window(tmp_path):
    from esm_b200 import extract_cli, windows
    path = _checkpoint(tmp_path)
    long_seq, short_seq = protein(150, 5), protein(30, 6)
    (tmp_path / "both.fasta").write_text(f">long\n{long_seq}\n>short\n{short_seq}\n")
    (tmp_path / "short.fasta").write_text(f">short\n{short_seq}\n")
    inc = ["--include", "mean", "per_tok", "bos", "--repr_layers", "0", "1", "-1"]
    p = extract_cli.create_parser()
    extract_cli.run(p.parse_args([path, str(tmp_path / "both.fasta"), str(tmp_path / "w")] + inc + ["--window", "62"]))
    extract_cli.run(p.parse_args([path, str(tmp_path / "short.fasta"), str(tmp_path / "plain")] + inc))
    a = torch.load(tmp_path / "w" / "short.pt")
    b = torch.load(tmp_path / "plain" / "short.pt")
    for key in ("representations", "mean_representations", "bos_representations"):
        assert sorted(a[key]) == sorted(b[key]) == [0, 1, 2]
        for layer in a[key]:
            assert torch.equal(a[key][layer], b[key][layer]), (key, layer)
    from esm_b200 import predict_cli
    from esm_b200.extract import mean_pool
    model, alphabet, _ = predict_cli.load_model(path)
    model = model.eval().cuda()
    _, _, tokens = alphabet.get_batch_converter()([("long", long_seq)])
    ref = model.forward_windowed(tokens.cuda(), 62, repr_layers=[0, 1, 2])["representations"]
    got = torch.load(tmp_path / "w" / "long.pt")
    for layer, t in ref.items():
        assert torch.equal(got["representations"][layer], t[0, 1:151].cpu())
        assert torch.equal(got["bos_representations"][layer], t[0, 0].cpu())
        m = mean_pool(t.contiguous(), torch.tensor([150], dtype=torch.int32, device="cuda"))[0].cpu()
        assert torch.equal(got["mean_representations"][layer], m)
    assert windows.starts(150, 62) == [0, 29, 58, 88]
