"""CPU: ESM-1b / ESM-1v (esm/model/esm1.py, arch roberta_large) host side — state-dict layout against the reference's
ProteinBertModel, the v1 checkpoint loader against the reference's own loader, the factories, the ESM-1 refusal, and
which reference layers patch_reference() dispatches.  The reference is imported from oracle/_ref (made by build())."""
import os
import sys
import warnings
from argparse import Namespace

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

from esm_b200 import ProteinBertModel, _lib, pretrained  # noqa: E402
from esm1b_weights import make_esm1b_state_dict  # noqa: E402  (tests/esm1b_weights.py)

ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")


@pytest.fixture(scope="module")
def esm_ref():
    if not os.path.isdir(os.path.join(REF, "esm")):
        pytest.fail("oracle/_ref/esm is missing: build() copies the reference there (oracle/reference.py)")
    sys.path.insert(0, REF)
    try:
        import esm  # the reference
        import esm.pretrained
        yield esm
    finally:
        sys.path.remove(REF)


def _args(L=2, E=128, H=2, ln_before=True, token_dropout=True):
    return Namespace(arch="roberta_large", layers=L, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                     max_positions=1024, emb_layer_norm_before=ln_before, token_dropout=token_dropout)


@pytest.mark.parametrize("ln_before", [True, False])
def test_state_dict_matches_reference_protein_bert_model(esm_ref, ln_before):
    args = _args(ln_before=ln_before)
    ref = esm_ref.ProteinBertModel(args, esm_ref.Alphabet.from_architecture("roberta_large"))
    ours = ProteinBertModel(args, "roberta_large")
    want = {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    got = {k: tuple(v.shape) for k, v in ours.state_dict().items()}
    assert got == want
    assert got["embed_positions.weight"] == (1024 + 1 + 1, 128)
    assert ("emb_layer_norm_before.weight" in got) == ln_before
    assert all("rot_emb" not in k for k in got)
    sd = make_esm1b_state_dict(2, 128, 2, emb_layer_norm_before=ln_before)
    assert set(sd) == set(want)
    ours.load_state_dict(sd, strict=True)
    assert ours.lm_head.weight is ours.embed_tokens.weight
    for k in ("num_layers", "alphabet_size", "padding_idx", "mask_idx", "cls_idx", "eos_idx", "prepend_bos",
              "append_eos", "model_version", "embed_scale"):
        assert getattr(ours, k) == getattr(ref, k), k
    # what BulkEmbedder / ShardedEmbedder / extract_cli read from a model
    assert (ours.embed_dim, ours.attention_heads, ours.alphabet.padding_idx) == (128, 2, 1)


def test_layer_without_rotary_matches_reference_esm1b_layer_keys(esm_ref):
    from esm_b200 import TransformerLayer
    ref = esm_ref.modules.TransformerLayer(128, 512, 2, add_bias_kv=False, use_esm1b_layer_norm=True)
    ours = TransformerLayer(128, 512, 2, use_rotary_embeddings=False)
    assert set(ours.state_dict()) == set(ref.state_dict())
    assert ours.self_attn.rot_emb is None
    assert "self_attn.rot_emb.inv_freq" in TransformerLayer(128, 512, 2).state_dict()  # ESM-2 layers unchanged


def _write_v1_checkpoint(path, sd, L, E, H, ln_before, with_regression):
    """The fairseq v1 layout the reference's loader reads (pretrained.py:85-101): Namespace args with encoder_ names,
    "encoder.sentence_encoder." / "encoder." parameter prefixes; the contact regression in a companion file."""
    args = Namespace(arch="roberta_large", encoder_layers=L, encoder_embed_dim=E, encoder_ffn_embed_dim=4 * E,
                     encoder_attention_heads=H, max_positions=1024, token_dropout=True)
    model = {}
    for k, v in sd.items():
        if k.startswith("contact_head.") or (k.startswith("emb_layer_norm_before") and not ln_before):
            continue
        prefix = "encoder." if k.startswith("lm_head.") else "encoder.sentence_encoder."
        model[prefix + k] = v  # lm_head.weight shares embed_tokens.weight's storage, as in the released files
    torch.save({"args": args, "model": model}, path)
    if with_regression:
        reg = {k: v.clone() for k, v in sd.items() if k.startswith("contact_head.")}
        torch.save({"model": reg}, str(path)[:-3] + "-contact-regression.pt")


@pytest.mark.parametrize("stem,ln_before,with_regression", [("esm1b_t2_tiny", True, True),
                                                            ("esm1v_t2_tiny_1", False, False)])
def test_v1_checkpoint_loads_like_the_reference_loader(esm_ref, tmp_path, stem, ln_before, with_regression):
    L, E, H = 2, 128, 2
    sd = make_esm1b_state_dict(L, E, H, seed=3, emb_layer_norm_before=ln_before)
    path = tmp_path / f"{stem}.pt"
    _write_v1_checkpoint(path, sd, L, E, H, ln_before, with_regression)
    with torch.serialization.safe_globals([Namespace]):  # the reference calls torch.load with the default weights_only
        with warnings.catch_warnings(record=True):
            warnings.simplefilter("always")
            ref, _ = esm_ref.pretrained.load_model_and_alphabet_local(str(path))
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        model, alphabet = pretrained.load_model_and_alphabet(str(path))
    assert isinstance(model, ProteinBertModel) and not model.random_init
    assert any("Regression weights not found" in str(x.message) for x in w) == (not with_regression)
    assert (model.emb_layer_norm_before is not None) == ln_before
    got, want = model.state_dict(), ref.state_dict()
    assert set(got) == set(want)
    for k in want:
        if k.startswith("contact_head.") and not with_regression:
            continue  # left at their initial values on both sides
        assert torch.equal(got[k], want[k]), k
    assert bool((got["embed_tokens.weight"][alphabet.mask_idx] == 0).all())  # zeroed for token dropout
    assert not bool((sd["embed_tokens.weight"][alphabet.mask_idx] == 0).all())


def test_v1_checkpoint_of_esm1_is_refused(tmp_path):
    torch.save({"args": Namespace(arch="protein_bert_base", decoder_layers=1), "model": {}}, tmp_path / "esm1_x.pt")
    with pytest.raises(ValueError, match="ESM-1"):
        pretrained.load_model_and_alphabet(str(tmp_path / "esm1_x.pt"))


def test_factories_raise_without_checkpoint_and_build_the_650M_shape(tmp_path, monkeypatch):
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    monkeypatch.delenv("ESMB200_ALLOW_RANDOM_INIT", raising=False)
    for fn in (pretrained.esm1b_t33_650M_UR50S, pretrained.esm1v_t33_650M_UR90S, pretrained.esm1v_t33_650M_UR90S_1,
               pretrained.esm1v_t33_650M_UR90S_2, pretrained.esm1v_t33_650M_UR90S_3, pretrained.esm1v_t33_650M_UR90S_4,
               pretrained.esm1v_t33_650M_UR90S_5):
        with pytest.raises(FileNotFoundError):
            fn()
    for name in pretrained.ESM1B_ARCH:
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            model, alphabet = pretrained.load_model_and_alphabet(name, allow_random_init=True, device="meta")
        assert model.random_init and any("RANDOM-INIT" in str(x.message) for x in w)
        assert isinstance(model, ProteinBertModel) and len(alphabet) == 33
        assert (model.num_layers, model.embed_dim, model.attention_heads) == (33, 1280, 20)
        assert model.layers[0].fc1.weight.shape == (5120, 1280)
        assert model.embed_positions.weight.shape == (1024 + 2, 1280) and model.embed_positions.max_positions == 1024
        assert model.emb_layer_norm_before is not None and model.token_dropout


@pytest.mark.parametrize("name", ["esm1_t34_670M_UR50S", "esm1_t34_670M_UR50D", "esm1_t34_670M_UR100",
                                  "esm1_t12_85M_UR50S", "esm1_t6_43M_UR50S"])
def test_esm1_names_raise(name):
    with pytest.raises(ValueError, match="ESM-1 \\(bias_kv attention\\) is not supported"):
        pretrained.load_model_and_alphabet(name, allow_random_init=True)
    with pytest.raises(ValueError, match="ESM-1 \\(bias_kv attention\\) is not supported"):
        getattr(pretrained, name)()
    with pytest.raises(ValueError):
        ProteinBertModel(Namespace(arch="protein_bert_base", layers=1, embed_dim=64, ffn_embed_dim=256,
                                   attention_heads=1, max_positions=1024), "roberta_large")


def test_forward_checks_length_first_and_has_no_cpu_fallback():
    model = ProteinBertModel(_args(L=1), "roberta_large").eval()
    with pytest.raises(ValueError, match="above maximum"):
        model(torch.zeros((1, 1025), dtype=torch.int64))
    with pytest.raises(_lib.Esmb200Error):
        model(torch.tensor([[0, 5, 6, 7, 2]]))


def test_patch_reference_dispatches_esm1b_layers_but_not_esm1(esm_ref):
    from esm_b200.integration import _dispatchable

    class _CudaLike:
        is_cuda = True

    M = esm_ref.modules
    esm1b = M.TransformerLayer(128, 512, 2, add_bias_kv=False, use_esm1b_layer_norm=True)
    esm1 = M.TransformerLayer(128, 512, 2, add_bias_kv=True, use_esm1b_layer_norm=False)
    esm2 = M.TransformerLayer(128, 512, 2, add_bias_kv=False, use_esm1b_layer_norm=True, use_rotary_embeddings=True)
    assert _dispatchable(esm1b, _CudaLike()) and _dispatchable(esm2, _CudaLike())
    assert not _dispatchable(esm1, _CudaLike())
    assert not _dispatchable(esm1b, torch.zeros(1))  # CPU tensors keep the reference path
