"""CPU: the streamed-weights ABI (esmb200_layer_packed_bytes, esmb200_layer_offload, esmb200_stack_forward_streamed) is
exported and its host arithmetic pinned; cpu_offload() refuses to run without a GPU before it moves anything; both
command lines take --cpu-offload, off by default."""
import ctypes

import pytest
import torch

NEW_SYMBOLS = ("esmb200_layer_packed_bytes", "esmb200_layer_offload", "esmb200_stack_forward_streamed")


def test_offload_symbols_are_exported_at_abi_version_4():
    from esm_b200 import _lib
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert name in _lib.EXPORTS
        assert hasattr(lib, name)
    assert _lib.load().esmb200_abi_version() == 4


@pytest.mark.parametrize("args,nbytes", [
    ((5120, 40, 20480, 0), 629_145_600),   # 15B: two 64-wide slots per 128-wide head
    ((2560, 40, 10240, 0), 157_286_400),   # 3B
    ((1280, 20, 5120, 0), 39_321_600),     # 650M
    ((320, 20, 1280, 0), 4_915_200),       # 8M: 16-wide heads padded to 64-wide slots
    ((1280, 20, 5120, 1), 2 * 39_321_600),  # fp32x3: hi | lo
    ((640, 20, 2560, 1), 2 * 13_107_200),
])
def test_packed_bytes_are_pinned(args, nbytes):
    from esm_b200 import _lib
    assert _lib.load().esmb200_layer_packed_bytes(*args) == nbytes


@pytest.mark.parametrize("args", [(0, 1, 64, 0), (512, 2, 2048, 0), (1280, 20, 0, 0), (1280, 20, 5120, 2),
                                  (1280, 3, 5120, 0)])
def test_packed_bytes_of_unsupported_shapes_are_zero(args):
    from esm_b200 import _lib
    assert _lib.load().esmb200_layer_packed_bytes(*args) == 0


def test_null_arguments_are_rejected_before_any_device_call():
    from esm_b200 import _lib
    lib = _lib.load()
    assert lib.esmb200_layer_offload(None, None, 0, None) == -1
    assert b"null" in lib.esmb200_last_error()
    assert lib.esmb200_stack_forward_streamed(None, 1, None, None, 1, 1, None, None, None, None, 0, 0, None, None, 0,
                                              None, 0, None, None) == -1
    assert b"null" in lib.esmb200_last_error()


@pytest.mark.parametrize("factory", ["esm2", "esm1b"])
def test_cpu_offload_without_a_gpu_raises_before_moving_anything(factory, monkeypatch):
    from esm_b200 import ESM2, _lib
    from esm_b200.esm1 import ProteinBertModel
    if factory == "esm2":
        model = ESM2(num_layers=2, embed_dim=128, attention_heads=2)
    else:
        model = ProteinBertModel(dict(layers=2, embed_dim=128, attention_heads=2, ffn_embed_dim=512,
                                      max_positions=64, emb_layer_norm_before=True))
    model.half()
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    before = {k: (v.device, v.dtype) for k, v in model.state_dict().items()}
    with pytest.raises(_lib.Esmb200Error):
        model.cpu_offload()
    assert {k: (v.device, v.dtype) for k, v in model.state_dict().items()} == before
    assert model._offload is None
    assert not any(layer.offloaded for layer in model.layers)


def test_cpu_offload_flag_parses_in_both_command_lines():
    from esm_b200 import extract_cli, predict_cli
    p = extract_cli.create_parser()
    base = ["esm2_t6_8M_UR50D", "in.fasta", "out", "--include", "mean"]
    assert p.parse_args(base).cpu_offload is False
    assert p.parse_args(base + ["--cpu-offload"]).cpu_offload is True
    assert p.parse_args(base).toks_per_batch == 65536
    q = predict_cli.create_parser()
    base = ["--model-location", "m.pt", "--sequence", "MK", "--dms-input", "a.csv", "--dms-output", "b.csv"]
    assert q.parse_args(base).cpu_offload is False
    assert q.parse_args(base + ["--cpu-offload"]).cpu_offload is True
