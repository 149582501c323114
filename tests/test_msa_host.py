"""CPU: host-side logic of the MSA Transformer mirror — state-dict layout, the checkpoint upgrade rule of
/root/reference/esm/pretrained.py:104-125 (fairseq prefixes stripped, "row" <-> "column" swapped, width of
msa_position_embedding taken from the tensor), constructor defaults, and the no-CPU-fallback contract."""
import ctypes
from argparse import Namespace

import pytest
import torch

from esm_b200 import pretrained
from esm_b200.alphabet import Alphabet
from esm_b200.msa import AxialTransformerLayer, MSATransformer


def small_args(**kw):
    d = dict(layers=2, embed_dim=128, ffn_embed_dim=256, attention_heads=2, max_positions=64, embed_positions_msa=True)
    d.update(kw)
    return Namespace(**d)


def test_state_dict_layout_matches_reference_names():
    m = MSATransformer(small_args())
    keys = set(m.state_dict().keys())
    for k in ("embed_tokens.weight", "msa_position_embedding", "embed_positions.weight",
              "emb_layer_norm_before.weight", "emb_layer_norm_after.bias", "lm_head.dense.weight", "lm_head.weight",
              "lm_head.bias", "lm_head.layer_norm.weight", "contact_head.regression.weight",
              "layers.0.row_self_attention.layer.q_proj.weight", "layers.1.column_self_attention.layer.out_proj.bias",
              "layers.0.row_self_attention.layer_norm.weight", "layers.1.feed_forward_layer.layer.fc1.weight",
              "layers.1.feed_forward_layer.layer_norm.bias"):
        assert k in keys, k
    assert m.state_dict()["embed_positions.weight"].shape == (64 + 1 + 1, 128)   # max_positions + padding_idx + 1
    assert m.state_dict()["msa_position_embedding"].shape == (1, 1024, 1, 128)
    assert m.state_dict()["contact_head.regression.weight"].shape == (1, 2 * 2)
    assert m.lm_head.weight is m.embed_tokens.weight                               # tied projection, modules.py:305


def test_checkpoint_upgrade_rule(tmp_path):
    """A checkpoint written the way the released esm_msa1*.pt files are laid out loads into the mirror."""
    ref = MSATransformer(small_args(embed_positions_msa_dim=1))       # first release: position width 1
    sd = ref.state_dict()

    def downgrade(k):  # inverse of the upgrade: swap row/column, add the fairseq prefixes
        k = k.replace("row", "column") if "row" in k else k.replace("column", "row")
        return "encoder.sentence_encoder." + k if not k.startswith("contact_head") else k

    model_part = {downgrade(k): v.clone() for k, v in sd.items() if not k.startswith("contact_head")}
    args = Namespace(arch="msa_transformer", encoder_layers=2, encoder_embed_dim=128, encoder_ffn_embed_dim=256,
                     encoder_attention_heads=2, max_positions=64, embed_positions_msa=True)
    path = tmp_path / "esm_msa_test.pt"
    torch.save({"args": args, "model": model_part}, str(path))
    torch.save({"model": {k: v for k, v in sd.items() if k.startswith("contact_head")}},
               str(tmp_path / "esm_msa_test-contact-regression.pt"))
    model, alphabet = pretrained.load_msa_model_and_alphabet(str(path))
    assert alphabet.use_msa and not model.random_init
    assert model.args.embed_positions_msa_dim == 1 and model.args.layers == 2
    got = model.state_dict()
    assert set(got.keys()) == set(sd.keys())
    for k in sd:
        assert torch.equal(got[k], sd[k]), k
    # the swap really happened: the file's "column" tensors are the mirror's "row" tensors
    assert torch.equal(model_part["encoder.sentence_encoder.layers.0.column_self_attention.layer.q_proj.weight"],
                       got["layers.0.row_self_attention.layer.q_proj.weight"])


def test_factories_return_model_and_msa_alphabet():
    model, alphabet = pretrained.esm_msa1b_t12_100M_UR50S(allow_random_init=True)
    assert isinstance(model, MSATransformer) and isinstance(alphabet, Alphabet)
    assert (model.args.layers, model.args.embed_dim, model.args.attention_heads) == (12, 768, 12)
    assert model.random_init and alphabet.prepend_bos and not alphabet.append_eos


def test_no_cpu_fallback_and_argument_checks():
    m = MSATransformer(small_args())
    tokens = torch.zeros(1, 2, 8, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(tokens)
    layer = AxialTransformerLayer(128, 256, 2)
    with pytest.raises(RuntimeError, match="CUDA"):
        layer(torch.zeros(2, 8, 1, 128))
    with pytest.raises(ValueError):
        AxialTransformerLayer(100, 256, 2)   # head_dim != 64


def test_factories_raise_without_checkpoint_unless_random_init_is_requested(tmp_path):
    """ADVICE r1: a missing checkpoint must not silently yield random weights (the reference fails when weights cannot
    be obtained, pretrained.py:53-64); strict key checking like pretrained.py:200-219."""
    import warnings
    from esm_b200 import ESM2
    with pytest.raises(FileNotFoundError):
        pretrained.esm2_t33_650M_UR50D()
    with pytest.raises(FileNotFoundError):
        pretrained.esm_msa1_t12_100M_UR50S()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        model, _ = pretrained.esm2_t6_8M_UR50D(allow_random_init=True)
    assert model.random_init and any("RANDOM-INIT" in str(x.message) for x in w)
    # a truncated checkpoint is an error, a checkpoint that only lacks the contact regression loads with a warning
    from oracle.weights import make_state_dict
    sd = make_state_dict(2, 128, 2)
    cfg = {"model": {"encoder_layers": 2, "encoder_embed_dim": 128, "encoder_attention_heads": 2, "token_dropout": True}}
    full = {("encoder.sentence_encoder." + k): v for k, v in sd.items()}
    torch.save({"cfg": cfg, "model": {k: v for k, v in full.items() if "layers.1.fc2" not in k}}, tmp_path / "bad.pt")
    with pytest.raises(RuntimeError, match="Missing key"):
        pretrained.load_model_and_alphabet(str(tmp_path / "bad.pt"))
    torch.save({"cfg": cfg, "model": {k: v for k, v in full.items() if "contact_head" not in k}}, tmp_path / "noreg.pt")
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        model, _ = pretrained.load_model_and_alphabet(str(tmp_path / "noreg.pt"))
    assert not model.random_init and any("Regression weights not found" in str(x.message) for x in w)
    torch.save({"cfg": cfg, "model": dict(full, **{"encoder.sentence_encoder.bogus": torch.zeros(1)})}, tmp_path / "extra.pt")
    with pytest.raises(RuntimeError, match="Unexpected key"):
        pretrained.load_model_and_alphabet(str(tmp_path / "extra.pt"))


# ---- argument refusals of the tied row attention: every check below returns before the device is touched -----------
# Placeholder pointers, which a refused call never dereferences; run only where no CUDA device is present, so that a
# refusal lost from the library can never turn into a launch on a bad address.  With a device,
# tests/test_gpu_tied_attention.py checks the same refusals with real buffers.
_FAKE = ctypes.c_void_p(4096)
no_device = pytest.mark.skipif(torch.cuda.is_available(), reason="placeholder pointers: only where nothing can launch")


@no_device
@pytest.mark.parametrize("split", [False, True], ids=["fp16", "fp32x3"])
@pytest.mark.parametrize("case,shape,rc,msg", [
    ("C=1025", (1, 1, 1025, 1), -1, b"1024"), ("BH=65536", (1024, 1, 1, 64), -1, b"bad shape"),
    ("H=65", (1, 1, 1, 65), -1, b"bad shape"), ("scratch-short", (2, 3, 5, 2), -4, b"scratch too small"),
    ("null-qkv", (2, 3, 5, 2), -1, b"null argument"), ("null-ctx", (2, 3, 5, 2), -1, b"null argument"),
    ("null-scratch", (2, 3, 5, 2), -1, b"null argument")])
def test_tied_row_attention_refusals(case, shape, rc, msg, split):
    from esm_b200 import _lib
    lib = _lib.load()
    B, R, C, H = shape
    nbytes = (lib.esmb200_tied_row_attention_split_scratch_bytes if split else
              lib.esmb200_tied_row_attention_scratch_bytes)(B, C, H)
    fn = lib.esmb200_tied_row_attention_split if split else lib.esmb200_tied_row_attention
    args = [_FAKE, None, _FAKE, None, B, R, C, H, _FAKE, nbytes - (case == "scratch-short"), None]
    if case.startswith("null"):
        args[{"null-qkv": 0, "null-ctx": 2, "null-scratch": 8}[case]] = None
    before = lib.esmb200_launch_count()
    assert fn(*args) == rc and msg in lib.esmb200_last_error(), lib.esmb200_last_error()
    assert lib.esmb200_launch_count() == before
