"""CPU: the fp32x3 precision mode of the MSA Transformer, everything that needs no device — MSATransformer.set_precision,
predict_cli --precision, the pinned sizes of the split stack workspace and tied scratch, and the split tied kernels in
the SASS of the shipped library."""
import os
import shutil
import subprocess
from argparse import Namespace

import pytest


def small_msa_model(layers=2, E=128, H=2):
    from esm_b200.msa import MSATransformer
    return MSATransformer(Namespace(layers=layers, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                                    max_positions=1024, embed_positions_msa=True))


def test_set_precision_validates_and_propagates():
    from esm_b200 import ESM2
    model = small_msa_model()
    assert model.precision == "fp16" and all(l.precision == 0 for l in model.layers)  # the default stays fp16
    assert model.PRECISIONS == ESM2.PRECISIONS == {"fp16": 0, "fp32x3": 1}
    assert model.set_precision("fp32x3") is model
    assert model.precision == "fp32x3" and all(l.precision == 1 for l in model.layers)
    model.set_precision("fp16")
    assert model.precision == "fp16" and all(l.precision == 0 for l in model.layers)
    for bad in ("fp32", "FP32X3", "", "bf16"):
        with pytest.raises(ValueError, match="precision must be one of"):
            model.set_precision(bad)
    assert model.precision == "fp16"  # a rejected name changes nothing


def test_predict_cli_precision_flag():
    from esm_b200 import predict_cli
    p = predict_cli.create_parser()
    base = ["--model-location", "m.pt", "--sequence", "MKT", "--dms-input", "in.csv", "--dms-output", "out.csv"]
    assert p.parse_args(base).precision == "fp16"
    assert p.parse_args(base + ["--precision", "fp32x3"]).precision == "fp32x3"
    opts = {a.dest: a for a in p._actions}
    assert opts["precision"].choices == ["fp16", "fp32x3"]
    with pytest.raises(SystemExit):
        p.parse_args(base + ["--precision", "fp32"])


class _StubModel:
    """Records what predict_cli.run does to a loaded model."""

    def __init__(self, calls):
        self.calls = calls

    def eval(self):
        return self

    def cuda(self):
        return self

    def set_precision(self, name):
        self.calls.append(name)
        return self


@pytest.mark.parametrize("flag,want", [([], []), (["--precision", "fp16"], []), (["--precision", "fp32x3"],
                                                                                   ["fp32x3", "fp32x3"])])
def test_predict_cli_applies_precision_to_every_model_location(flag, want, tmp_path, monkeypatch):
    from esm_b200 import predict_cli
    calls = []
    monkeypatch.setattr(predict_cli, "load_model", lambda loc: (_StubModel(calls), None, loc == "msa.pt"))
    monkeypatch.setattr(predict_cli, "score_model", lambda model, alphabet, is_msa, args, muts: [0.5] * len(muts))
    dms = tmp_path / "dms.csv"
    dms.write_text("mutant\nM1A\nK2R\n")
    out = tmp_path / "out.csv"
    args = predict_cli.create_parser().parse_args(["--model-location", "seq.pt", "msa.pt", "--sequence", "MKT",
                                                   "--dms-input", str(dms), "--dms-output", str(out)] + flag)
    predict_cli.run(args)
    assert calls == want
    assert out.read_text() == ",mutant,seq.pt,msa.pt\n0,M1A,0.5,0.5\n1,K2R,0.5,0.5\n"


@pytest.mark.parametrize("fn,args,nbytes", [
    ("esmb200_axial_workspace_bytes_split", (768, 3072, 1, 128, 512), 1038104576),
    ("esmb200_axial_workspace_bytes_split", (128, 512, 2, 5, 130), 4029440),
    ("esmb200_axial_workspace_bytes_split", (256, 1024, 3, 7, 61), 6974720),
    ("esmb200_tied_row_attention_split_scratch_bytes", (1, 512, 12), 25167872),
    ("esmb200_tied_row_attention_split_scratch_bytes", (2, 130, 4), 1342464),
    ("esmb200_tied_row_attention_split_scratch_bytes", (1, 64, 2), 67584),
])
def test_split_workspace_sizes_are_pinned(fn, args, nbytes):
    """The split stack holds every fp16 activation (LayerNorm output, qkv, ctx, FFN hidden) and P as hi | lo pairs:
    those parts double; the key bits, row statistics and fp32 logits do not."""
    from esm_b200 import _lib
    assert getattr(_lib.load(), fn)(*args) == nbytes


def test_split_tied_scratch_doubles_only_p():
    from esm_b200 import _lib
    lib = _lib.load()
    for B, C, H in [(1, 512, 12), (2, 130, 4), (3, 1000, 2)]:
        f16 = lib.esmb200_tied_row_attention_scratch_bytes(B, C, H)
        split = lib.esmb200_tied_row_attention_split_scratch_bytes(B, C, H)
        Cp = (C + 63) // 64 * 64
        p_bytes = (H * B * C * Cp * 2 + 1023) // 1024 * 1024
        assert split - f16 == p_bytes


def test_split_tied_kernels_run_on_the_tensor_cores():
    """Both instances of the tied logits / update kernels use the warp-level tensor-core MMA (HMMA)."""
    from esm_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump) or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or the built library is not available")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    hmma, cur = {}, None
    for line in sass.splitlines():
        if "Function :" in line:
            cur = line.split("Function :")[1].strip()
            hmma[cur] = 0
        elif cur and "HMMA" in line:
            hmma[cur] += 1
    for kernel in ("tied_scores_kernel", "tied_pv_kernel"):
        for inst in ("ILb0E", "ILb1E"):
            found = [n for n in hmma if kernel in n and inst in n]
            assert len(found) == 1 and hmma[found[0]] > 0, (kernel, inst, found)
    # the split update runs three products per fp16 one
    pv = {i: hmma[[n for n in hmma if "tied_pv_kernel" in n and i in n][0]] for i in ("ILb0E", "ILb1E")}
    assert pv["ILb1E"] == 3 * pv["ILb0E"]
