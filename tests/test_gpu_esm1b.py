"""GPU (-m gpu): ESM-1b / ESM-1v (esm_b200.ProteinBertModel) on the sm_90a kernels.

  * esmb200_esm1b_embed against a PyTorch restatement of esm/model/esm1.py:123-139;
  * the model against committed outputs of the unmodified reference ProteinBertModel (tests/golden/esm1b_*.pt, made by
    tests/golden/make_golden_esm1b.py) at the ESM-2 tolerances of DESIGN.md section 4;
  * full size (33 x 1280 x 20 heads, T = 1024) against the reference run eager fp32 on the same GPU;
  * the reference's own ProteinBertModel patched onto the library (INTEGRATION.md Option B);
  * fp32x3, model.half(), the position-table limit, and the extraction CLI.
"""
import argparse
import ctypes
import os
import sys

import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # esm1b_weights (tests/esm1b_weights.py)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
FIXTURES = ["esm1b_tiny_L2_E128_H2", "esm1b_mid_L3_E256_H4", "esm1b_edge_L1_E128_H2_T1024"]

REL_FRO = 3e-3
REL_FRO_LOGITS = 4e-3
ATT_ABS = 1e-2
CONTACT_ABS = 1e-2


def rel_fro(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def checksum(sd):
    return float(sum(v.double().abs().sum() for k, v in sorted(sd.items())))


@pytest.fixture(scope="module")
def esm_ref():
    if not os.path.isdir(os.path.join(REF, "esm")):
        pytest.fail("oracle/_ref/esm is missing: build() copies the reference there (oracle/reference.py)")
    sys.path.insert(0, REF)
    try:
        import esm  # the reference
        import esm.modules
        yield esm
    finally:
        sys.path.remove(REF)


# ---- the embedding kernel -----------------------------------------------------------------------------------------
def embed_torch(tokens, table, pos_table, ln_w, ln_b, token_dropout, padding_idx=1, mask_idx=32):
    """esm1.py:121-139 + LearnedPositionalEmbedding.forward (modules.py:240-257), fp32 on the same device."""
    padding_mask = tokens.eq(padding_idx)
    x = F.embedding(tokens, table)
    if token_dropout:
        x.masked_fill_((tokens == mask_idx).unsqueeze(-1), 0.0)
        src_lengths = (~padding_mask).sum(-1)
        ratio = (tokens == mask_idx).sum(-1).float() / src_lengths
        x = x * (1 - 0.15 * 0.8) / (1 - ratio)[:, None, None]
    mask = tokens.ne(padding_idx).int()
    positions = (torch.cumsum(mask, dim=1).type_as(mask) * mask).long() + padding_idx
    x = x + F.embedding(positions, pos_table)
    if ln_w is not None:
        x = F.layer_norm(x, (x.shape[-1],), ln_w, ln_b, 1e-5)
    return x * (1 - padding_mask.unsqueeze(-1).type_as(x))


def embed_lib(tokens, table, pos_table, ln_w, ln_b, token_dropout, padding_idx=1, mask_idx=32):
    from esm_b200 import _lib
    from esm_b200.model import _ptr, _stream
    B, T = tokens.shape
    E = table.shape[1]
    x = torch.full((B, T, E), float("nan"), device="cuda")
    _lib.check(_lib.load().esmb200_esm1b_embed(_ptr(tokens), _ptr(table), _ptr(pos_table), _ptr(ln_w), _ptr(ln_b),
                                               1e-5, int(token_dropout), padding_idx, mask_idx, _ptr(x), B, T, E,
                                               _stream()))
    return x


@pytest.mark.parametrize("E", [1280, 320, 2560])
@pytest.mark.parametrize("token_dropout", [True, False])
@pytest.mark.parametrize("ln", [True, False])
@pytest.mark.parametrize("T", [77, 1024])
def test_embed_kernel_matches_torch(E, token_dropout, ln, T):
    g = torch.Generator().manual_seed(E + T + 2 * token_dropout + ln)
    B = 5
    tokens = torch.randint(4, 24, (B, T), generator=g)
    tokens[:, 0] = 0
    lengths = [T - 2, T // 2, 3, T - 9, T - 2]
    for b, n in enumerate(lengths):
        tokens[b, n + 1] = 2
        tokens[b, n + 2:] = 1
    tokens[0, 3] = tokens[0, 7] = tokens[3, T // 3] = 32      # <mask>
    tokens[1, 5] = tokens[4, 2] = tokens[4, T - 40] = 1        # <pad> inside a sequence
    tokens = tokens.cuda()
    table = torch.randn(33, E, generator=g).cuda()
    pos_table = torch.randn(1024 + 2, E, generator=g).cuda()
    ln_w = (1 + 0.2 * torch.randn(E, generator=g)).cuda() if ln else None
    ln_b = (0.1 * torch.randn(E, generator=g)).cuda() if ln else None
    got = embed_lib(tokens, table, pos_table, ln_w, ln_b, token_dropout)
    want = embed_torch(tokens, table, pos_table, ln_w, ln_b, token_dropout)
    assert float((got - want).abs().max()) <= 1e-5


def test_embed_and_stack_argument_checks():
    from esm_b200 import ProteinBertModel, _lib
    from esm_b200.model import _ptr, _stream, _workspace
    lib = _lib.load()
    tok = torch.zeros((1, 8), dtype=torch.int64, device="cuda")
    table, x = torch.zeros((33, 128), device="cuda"), torch.zeros((1, 8, 128), device="cuda")
    w = torch.ones(128, device="cuda")
    # LayerNorm weight without bias
    assert lib.esmb200_esm1b_embed(_ptr(tok), _ptr(table), _ptr(table), _ptr(w), None, 1e-5, 0, 1, 32, _ptr(x), 1, 8,
                                   128, _stream()) == -1
    # exactly one rotary table is an error; none is the ESM-1b layer
    model = ProteinBertModel(argparse.Namespace(arch="roberta_large", layers=1, embed_dim=128, ffn_embed_dim=512,
                                                attention_heads=2, max_positions=1024), "roberta_large").cuda()
    h = model.layers[0].handle()
    nbytes = lib.esmb200_workspace_bytes(128, 2, 512, 1, 8, 0)
    ws = _workspace(nbytes, x.device)
    cos = torch.ones((8, 32), device="cuda")
    handles = (ctypes.c_void_p * 1)(h)
    for c, s in ((cos, None), (None, cos)):
        assert lib.esmb200_layer_forward(h, _ptr(x), None, 1, 8, _ptr(c), _ptr(s), None, _ptr(ws), ws.numel(),
                                         _stream()) == -1
        assert lib.esmb200_stack_forward(handles, 1, _ptr(x), None, 1, 8, _ptr(c), _ptr(s), None, None, 0, 0, None,
                                         _ptr(ws), ws.numel(), _stream()) == -1
    assert lib.esmb200_layer_forward(h, _ptr(x), None, 1, 8, None, None, None, _ptr(ws), ws.numel(), _stream()) == 0
    torch.cuda.synchronize()


# ---- the model against the reference's committed outputs ----------------------------------------------------------
def build_model(fx, precision="fp16"):
    from esm_b200 import ProteinBertModel
    from esm1b_weights import make_esm1b_state_dict
    cfg = fx["config"]
    args = argparse.Namespace(**cfg["model_args"])
    sd = make_esm1b_state_dict(cfg["num_layers"], cfg["embed_dim"], cfg["attention_heads"], seed=cfg["seed"],
                               emb_layer_norm_before=args.emb_layer_norm_before)
    assert abs(checksum(sd) - fx["state_dict_checksum"]) <= 1e-6 * fx["state_dict_checksum"]
    model = ProteinBertModel(args, "roberta_large")
    model.load_state_dict(sd, strict=True)
    return model.eval().cuda().set_precision(precision), sd


def stored(out, fx):
    """The library's outputs cut to what the fixture stores: token positions fx["rows"] (the whole sequence for all but
    the T = 1024 case), the attention sub-sample and the contact rows fx["contacts_rows"]."""
    r0, r1 = fx["rows"]
    c0, c1 = fx["contacts_rows"]
    res = {"logits": out["logits"][:, r0:r1].float().cpu(),
           "representations": {k: v[:, r0:r1].float().cpu() for k, v in out["representations"].items()}}
    if "attentions" in out:
        sub = out["attentions"][:, fx["attentions_sub_layers"]][:, :, fx["attentions_sub_heads"]]
        res["attentions_sub"] = sub[..., r0:r1, :].float().cpu()
    if "contacts" in out:
        res["contacts"] = out["contacts"][:, c0:c1].float().cpu()
    return res


def check_against_fixture(out, fx, rel=REL_FRO, rel_logits=REL_FRO_LOGITS, att=ATT_ABS, contact=CONTACT_ABS):
    got = stored(out, fx)
    for k, ref in fx["representations"].items():
        assert got["representations"][k].shape == ref.shape
        assert rel_fro(got["representations"][k], ref) <= rel, (k, rel_fro(got["representations"][k], ref))
    assert rel_fro(got["logits"], fx["logits"]) <= rel_logits
    assert float((got["attentions_sub"] - fx["attentions_sub"]).abs().max()) <= att
    c = float((got["contacts"] - fx["contacts"]).abs().max())
    assert c <= contact, c


@pytest.mark.parametrize("name", FIXTURES)
def test_against_reference_golden(name, golden_dir):
    fx = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    model, _ = build_model(fx)
    out = model(fx["tokens"].cuda(), repr_layers=fx["repr_layers"], need_head_weights=True, return_contacts=True)
    torch.cuda.synchronize()
    assert set(out.keys()) == {"logits", "representations", "attentions", "contacts"}
    check_against_fixture(out, fx)
    # the same representations without attention maps (the probability pass is skipped)
    L = fx["config"]["num_layers"]
    plain = model(fx["tokens"].cuda(), repr_layers=[L])
    assert torch.equal(plain["representations"][L], out["representations"][L])


def test_fp32x3_against_reference_golden(golden_dir):
    """the bound tests/test_gpu_precision.py holds ESM-2's fp32x3 mode to"""
    fx = torch.load(os.path.join(golden_dir, "esm1b_mid_L3_E256_H4.pt"), weights_only=False)
    model, _ = build_model(fx, "fp32x3")
    out = model(fx["tokens"].cuda(), repr_layers=fx["repr_layers"], return_contacts=True)
    torch.cuda.synchronize()
    k = fx["config"]["num_layers"]
    got = stored(out, fx)
    r = rel_fro(got["representations"][k], fx["representations"][k])
    lg = rel_fro(got["logits"], fx["logits"])
    c = float((got["contacts"] - fx["contacts"]).abs().max())
    print(f"PARITY fp32x3 esm1b_mid_L3_E256_H4: repr rel_fro={r:.3e} logits={lg:.3e} contacts max_abs={c:.3e}")
    assert r <= 2e-5 and lg <= 2e-5 and c <= 1e-4


def test_half_model_returns_fp16_and_length_limit(golden_dir):
    fx = torch.load(os.path.join(golden_dir, "esm1b_tiny_L2_E128_H2.pt"), weights_only=False)
    model, _ = build_model(fx)
    model = model.half()
    out = model(fx["tokens"].cuda(), repr_layers=fx["repr_layers"], return_contacts=True)
    assert out["logits"].dtype == torch.float16 and out["contacts"].dtype == torch.float16
    assert all(v.dtype == torch.float16 for v in out["representations"].values())
    L = fx["config"]["num_layers"]
    # fp16-rounded weights on both the position table and the layers: within the fp16 model tolerance
    assert rel_fro(stored(out, fx)["representations"][L], fx["representations"][L]) <= 8e-3
    with pytest.raises(ValueError, match="above maximum"):
        model(torch.zeros((1, 1025), dtype=torch.int64, device="cuda"))


# ---- full size against the reference, eager fp32 on the same GPU ---------------------------------------------------
def test_reference_esm1b_650M_full_size_eager_vs_library(esm_ref):
    from esm_b200 import ProteinBertModel
    from esm1b_weights import make_esm1b_state_dict
    from oracle.weights import make_tokens
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    L, E, H = 33, 1280, 20
    args = argparse.Namespace(arch="roberta_large", layers=L, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                              max_positions=1024, emb_layer_norm_before=True, token_dropout=True)
    sd = make_esm1b_state_dict(L, E, H, seed=0)
    tokens = make_tokens([1022, 700], 1024, seed=4, n_mask=3).cuda()
    ref = esm_ref.ProteinBertModel(args, esm_ref.Alphabet.from_architecture("roberta_large"))
    ref.load_state_dict(sd, strict=True)
    ref = ref.eval().cuda()
    with torch.no_grad():
        eager = ref(tokens, repr_layers=[L], return_contacts=True)
        eager = {"rep": eager["representations"][L], "logits": eager["logits"], "contacts": eager["contacts"]}
    del ref
    model = ProteinBertModel(args, "roberta_large")
    model.load_state_dict(sd, strict=True)
    model = model.eval().cuda()
    fast = model(tokens, repr_layers=[L], return_contacts=True)
    keep = tokens.ne(1)
    r = rel_fro(fast["representations"][L][keep], eager["rep"][keep])
    rl = rel_fro(fast["logits"][keep], eager["logits"][keep])
    rc = float((fast["contacts"] - eager["contacts"])[0].abs().max())  # sequence 0 has no padding
    print(f"PARITY reference_eager_esm1b_650M_T1024 repr={r:.3e} logits={rl:.3e} contacts_abs={rc:.3e}", flush=True)
    assert r <= REL_FRO and rl <= REL_FRO_LOGITS and rc <= CONTACT_ABS


# ---- Option B: the reference's own ProteinBertModel with its layers on the library ---------------------------------
def _reference_from_fixture(esm, fx):
    from esm1b_weights import make_esm1b_state_dict
    cfg = fx["config"]
    args = argparse.Namespace(**cfg["model_args"])
    sd = make_esm1b_state_dict(cfg["num_layers"], cfg["embed_dim"], cfg["attention_heads"], seed=cfg["seed"],
                               emb_layer_norm_before=args.emb_layer_norm_before)
    model = esm.ProteinBertModel(args, esm.Alphabet.from_architecture("roberta_large"))
    model.load_state_dict(sd, strict=True)
    return model.eval()


@pytest.mark.parametrize("name", FIXTURES[:2])
def test_patched_reference_esm1b_on_the_library(esm_ref, name, golden_dir):
    from esm_b200 import _lib, integration
    fx = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    model = _reference_from_fixture(esm_ref, fx).cuda()
    integration.patch_reference(esm_ref.modules)
    try:
        n0 = _lib.load().esmb200_launch_count()
        with torch.no_grad():
            out = model(fx["tokens"].cuda(), repr_layers=fx["repr_layers"], need_head_weights=True,
                        return_contacts=True)
        torch.cuda.synchronize()
        launched = _lib.load().esmb200_launch_count() - n0
    finally:
        integration.unpatch_reference(esm_ref.modules)
    assert launched >= 7 * fx["config"]["num_layers"], "the reference's layers did not go through libesmb200.so"
    check_against_fixture(out, fx)


def test_patched_reference_esm1b_keeps_cpu_tensors_on_the_reference_path(esm_ref, golden_dir):
    """Bit-identical to the unpatched reference on CPU tensors, and nothing is launched on the library.  One CPU thread:
    with several, the host BLAS may split its sums differently from one call to the next (MKL's dynamic threading
    picks the thread count per call), so two runs of the UNPATCHED reference can already differ in the last bit; the
    first call of a shape is also left out of the comparison."""
    from esm_b200 import _lib, integration
    fx = torch.load(os.path.join(golden_dir, "esm1b_tiny_L2_E128_H2.pt"), weights_only=False)
    model = _reference_from_fixture(esm_ref, fx)
    tokens = fx["tokens"][:, :20].clone()
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        with torch.no_grad():
            model(tokens, repr_layers=[2], return_contacts=True)  # first call of each shape: kernel selection
            want = model(tokens, repr_layers=[2], return_contacts=True)
        integration.patch_reference(esm_ref.modules)
        try:
            n0 = _lib.load().esmb200_launch_count()
            with torch.no_grad():
                got = model(tokens, repr_layers=[2], return_contacts=True)
            assert _lib.load().esmb200_launch_count() == n0
        finally:
            integration.unpatch_reference(esm_ref.modules)
    finally:
        torch.set_num_threads(threads)
    for k in ("logits", "contacts", "attentions"):
        assert torch.equal(got[k], want[k]), k
    assert torch.equal(got["representations"][2], want["representations"][2])


# ---- extraction ------------------------------------------------------------------------------------------------------
def test_extract_cli_on_an_esm1b_checkpoint(tmp_path):
    from esm_b200 import extract_cli, pretrained
    from esm1b_weights import make_esm1b_state_dict
    L, E, H = 2, 128, 2
    sd = make_esm1b_state_dict(L, E, H, seed=5)
    args = argparse.Namespace(arch="roberta_large", encoder_layers=L, encoder_embed_dim=E,
                              encoder_ffn_embed_dim=4 * E, encoder_attention_heads=H, max_positions=1024,
                              token_dropout=True)
    model_sd = {("encoder." if k.startswith("lm_head.") else "encoder.sentence_encoder.") + k: v
                for k, v in sd.items() if not k.startswith("contact_head.")}
    ckpt = tmp_path / "esm1b_tiny.pt"
    torch.save({"args": args, "model": model_sd}, ckpt)
    torch.save({"model": {k: v for k, v in sd.items() if k.startswith("contact_head.")}},
               tmp_path / "esm1b_tiny-contact-regression.pt")
    fasta = tmp_path / "in.fasta"
    seqs = {"p1": "MKTVRQERLKSIVRILERSKEPVSGAQ", "p2": "KALTARQQEVFDLIRD", "p3": "MKT"}
    fasta.write_text("".join(f">{k}\n{v}\n" for k, v in seqs.items()))
    outdir = tmp_path / "out"
    cli = argparse.Namespace(model_location=str(ckpt), fasta_file=fasta, output_dir=outdir, toks_per_batch=64,
                             repr_layers=[-1], include=["mean", "per_tok", "bos", "contacts"],
                             truncation_seq_length=1022, precision="fp16")
    assert extract_cli.run(cli) == 3
    model, alphabet = pretrained.load_model_and_alphabet(str(ckpt))
    model = model.cuda()
    for label, seq in seqs.items():
        r = torch.load(outdir / f"{label}.pt", weights_only=False)
        assert set(r.keys()) == {"label", "representations", "mean_representations", "bos_representations", "contacts"}
        _, _, tok = alphabet.get_batch_converter()([(label, seq)])
        direct = model(tok.cuda(), repr_layers=[L], return_contacts=True)
        rep = direct["representations"][L][0].cpu()
        torch.testing.assert_close(r["representations"][L], rep[1:len(seq) + 1], atol=1e-5, rtol=1e-5)
        torch.testing.assert_close(r["mean_representations"][L], rep[1:len(seq) + 1].mean(0), atol=1e-5, rtol=1e-5)
        torch.testing.assert_close(r["bos_representations"][L], rep[0], atol=1e-5, rtol=1e-5)
        torch.testing.assert_close(r["contacts"], direct["contacts"][0].cpu(), atol=1e-5, rtol=1e-5)
