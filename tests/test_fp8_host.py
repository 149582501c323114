"""CPU: the fp8 precision, everything that needs no device — the scale rule and e4m3 rounding of the torch reference the
GPU tests compare the kernels with, set_precision("fp8") on every model shape, the pinned workspace size, the offload
refusals, extract_cli --precision fp8, and the fp8 GEMM in the SASS of the shipped library."""
import os
import shutil
import subprocess
from argparse import Namespace

import pytest
import torch

import fp8_refs as fr


def test_scale_is_the_smallest_power_of_two():
    assert fr.block_scale(0.0) == 1.0                       # all-zero block
    assert fr.block_scale(448.0) == 1.0                     # the exact amax: 448 / 1 <= 448
    assert fr.block_scale(448.0 * (1 + 2 ** -20)) == 2.0    # just above it
    assert fr.block_scale(1.0) == 2.0 ** -8                 # 256 <= 448 < 512
    assert fr.block_scale(1.75) == 2.0 ** -8 and fr.block_scale(1.76) == 2.0 ** -7
    assert fr.block_scale(1e-40) == 2.0 ** -126             # never below the smallest normal float
    for a in torch.rand(200, dtype=torch.float64) * 1e4:
        s = fr.block_scale(float(a))
        assert a / s <= 448 < a / (s / 2)
    amax = torch.tensor([0.0, 448.0, 449.0, 1.0, 1e-40, 3.5e7])
    assert [fr.block_scale(float(a)) for a in amax] == fr.scales_of(amax).tolist()


def test_quantize_rounds_to_nearest_even_and_keeps_signs():
    x = torch.zeros(2, 256)
    x[0, 0] = 448.0                      # scale 1
    x[0, 1] = -17.0                      # between 16 and 18: a tie, rounds to the even code 16
    x[0, 2] = -19.0                      # tie between 18 and 20: 20
    x[0, 3] = 2.0 ** -9                  # the smallest e4m3 subnormal at scale 1
    x[0, 4] = 2.0 ** -11                 # half of it: rounds to zero (even)
    x[0, 5] = 3 * 2.0 ** -10             # tie between 2^-9 and 2^-8: the even code 2^-8
    q, s = fr.quantize(x, 1)
    assert s.shape == (2, 2) and s[0, 0] == 1.0 and s[1, 0] == 1.0  # block 1 of row 0 and row 1: all zero
    d = q.float()[0, :6].tolist()
    assert d == [448.0, -16.0, -20.0, 2.0 ** -9, 0.0, 2.0 ** -8]


def test_partial_blocks_take_their_scale_over_valid_columns():
    x = torch.zeros(130, 320)
    x[:, 256:] = 3.0                     # the partial third K block (64 valid columns)
    x[129, 5] = 900.0                    # a weight block of 2 valid rows
    q, s = fr.quantize(x, 1)
    assert s.shape == (3, 130) and bool((s[2] == 2.0 ** -7).all()) and bool((s[:2, :129] == 1).all())
    qw, sw = fr.quantize(x, 128)
    assert sw.shape == (2, 3) and sw[1, 0] == 4.0 and sw[0, 2] == 2.0 ** -7
    back = fr.dequantize(q, s, 1)
    assert torch.equal(back[:, 256:].float(), x[:, 256:])


def _layer_shapes():
    # (num_layers, embed_dim, heads): every esm2_* size's layer shape, ESM-1b / 1v's
    return [(1, 320, 20), (1, 480, 20), (1, 640, 20), (1, 1280, 20), (1, 2560, 40), (1, 5120, 40)]


@pytest.mark.parametrize("L,E,H", _layer_shapes())
def test_set_precision_fp8_on_every_esm2_shape(L, E, H):
    from esm_b200 import ESM2
    with torch.device("meta"):
        model = ESM2(num_layers=L, embed_dim=E, attention_heads=H)
    model.set_precision("fp8")
    assert model.precision == "fp8" and all(layer.precision == 2 for layer in model.layers)
    assert model._lm_head_precision() == 0  # the fp8 mode's LM head runs fp16
    model.set_precision("fp16")
    assert all(layer.precision == 0 for layer in model.layers)


def test_set_precision_fp8_on_esm1b():
    from esm_b200 import ProteinBertModel
    args = Namespace(arch="roberta_large", layers=1, embed_dim=128, ffn_embed_dim=512, attention_heads=2,
                     max_positions=1024, token_dropout=True, emb_layer_norm_before=True)
    model = ProteinBertModel(args, "roberta_large")
    model.set_precision("fp8")
    assert model.layers[0].precision == 2


def test_msa_transformer_refuses_fp8():
    from esm_b200.msa import MSATransformer
    m = MSATransformer(Namespace(layers=1, embed_dim=128, ffn_embed_dim=512, attention_heads=2, max_positions=1024,
                                 embed_positions_msa=True))
    with pytest.raises(ValueError):
        m.set_precision("fp8")


@pytest.mark.parametrize("args,nbytes", [
    ((1280, 20, 5120, 256, 1024), 3072362496),   # 650M, the bulk-embedding batch
    ((320, 20, 1280, 2, 100), 2149376),          # 8M: partial K blocks (E = 320)
    ((480, 20, 1920, 3, 77), 2521088),           # 35M
    ((5120, 40, 20480, 1, 1024), 47678976),      # 15B: two-slot heads
])
def test_fp8_workspace_bytes_are_pinned(args, nbytes):
    from esm_b200 import _lib
    lib = _lib.load()
    assert lib.esmb200_workspace_bytes(*args, 2) == nbytes
    assert lib.esmb200_layer_packed_bytes(args[0], args[1], args[2], 2) == 0  # fp8 layers are not streamed


def test_cpu_offload_refuses_fp8():
    from esm_b200 import ESM2, _lib
    model = ESM2(num_layers=1, embed_dim=64, attention_heads=2).set_precision("fp8")
    with pytest.raises(_lib.Esmb200Error, match="fp8"):
        model.cpu_offload()
    model.set_precision("fp16")
    model._offload = ("cuda:0", None)  # an offloaded model (cpu_offload() needs a device)
    with pytest.raises(_lib.Esmb200Error, match="fp8"):
        model.set_precision("fp8")
    assert model.precision == "fp16" and model.layers[0].precision == 0
    model._offload = None


def test_extract_cli_parses_fp8():
    from esm_b200.extract_cli import create_parser
    a = create_parser().parse_args(["esm2_t6_8M_UR50D", "x.fasta", "out", "--include", "mean", "--precision", "fp8"])
    assert a.precision == "fp8"


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"),
                    reason="cuobjdump not available")
def test_fp8_gemm_runs_e4m3_wgmma_without_spills():
    from esm_b200 import _lib
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([exe, "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    for epi in (0, 1, 5):
        name = f"gemm_fp8_e4m3_kernelILi{epi}E"
        i = sass.index(name)
        j = sass.find("Function :", i)
        body = sass[i:j if j > 0 else None]
        assert body.count("QGMMA.64x128x32.F32.E4M3.E4M3") == 4
        assert "LDL" not in body and "STL" not in body
    assert sass.count("gemm2_f16_kernel") >= 10
