"""CPU: the C-ABI library builds, loads and exports exactly what include/esmb200.h declares; the product package
never touches the oracle; the product path fails loudly without a GPU (no CPU fallback)."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "esmb200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(esmb200_[a-z0-9_]+)\s*\(", text)))


def test_library_builds_and_exports_every_declared_symbol_at_abi_version_4():
    from esm_b200 import _lib, build
    path = build.build()
    assert os.path.exists(path)
    lib = ctypes.CDLL(path)
    declared = header_symbols()
    assert declared, "no symbols parsed from the header"
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/esmb200.h but not exported"
    assert sorted(_lib.EXPORTS) == declared
    assert _lib.load().esmb200_abi_version() == 4


def test_workspace_size_is_pure_host_arithmetic():
    from esm_b200 import _lib
    lib = _lib.load()
    small = lib.esmb200_workspace_bytes(1280, 20, 5120, 1, 1024, 0)
    big = lib.esmb200_workspace_bytes(1280, 20, 5120, 256, 1024, 0)
    assert 0 < small < big
    assert big >= 256 * 1024 * (1280 * 2 + 5120 * 2)  # xn + h
    assert lib.esmb200_workspace_bytes(1280, 20, 5120, 256, 1024, 1) >= 2 * 256 * 1024 * (1280 * 2 + 5120 * 2)  # fp32x3


@pytest.mark.parametrize("fn,args,nbytes", [
    ("esmb200_workspace_bytes", (1280, 20, 5120, 256, 1024, 0), 3397421056),
    ("esmb200_workspace_bytes", (1280, 20, 5120, 256, 1024, 1), 6752864256),
    ("esmb200_workspace_bytes", (320, 20, 1280, 3, 1003, 0), 33222912),       # head_dim 16, odd T
    ("esmb200_workspace_bytes", (5120, 40, 20480, 16, 1024, 0), 844107008),   # head_dim 128: two slots per head
    ("esmb200_workspace_bytes", (2560, 40, 10240, 16, 512, 0), 212338944),
    ("esmb200_workspace_bytes", (640, 20, 2560, 5, 77, 1), 8934400),
    ("esmb200_axial_workspace_bytes", (768, 3072, 1, 128, 512), 528496640),
    ("esmb200_axial_workspace_bytes", (128, 512, 2, 5, 130), 2165760),
    ("esmb200_axial_workspace_bytes", (256, 1024, 3, 7, 61), 3603712),
    ("esmb200_attention_scratch_bytes", (2, 1024), 1049088),
    ("esmb200_attention_scratch_bytes", (33, 77), 1302016),
    ("esmb200_tied_row_attention_scratch_bytes", (1, 512, 12), 18876416),
    ("esmb200_tied_row_attention_scratch_bytes", (2, 130, 4), 943104),
])
def test_workspace_layout_is_pinned(fn, args, nbytes):
    """Exact sizes of every workspace / scratch layout: callers allocate from these, so a layout change shows here."""
    from esm_b200 import _lib
    assert getattr(_lib.load(), fn)(*args) == nbytes


def test_product_package_never_imports_the_oracle():
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "esm_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M) or "oracle/" in src:
                    bad.append(os.path.join(dirpath, f))
    assert not bad, f"product code references the oracle: {bad}"


def test_no_cpu_fallback():
    from esm_b200 import ESM2, _lib
    model = ESM2(num_layers=1, embed_dim=128, attention_heads=2).eval()
    tokens = torch.tensor([[0, 5, 6, 7, 2]])
    with pytest.raises(_lib.Esmb200Error):
        model(tokens)


def test_every_esm2_factory_shape_constructs():
    """esm.pretrained.esm2_* (pretrained.py:344-397): head_dim 16 / 24 / 32 / 64 / 128 construct (heads that are not 64
    wide run in padded 64-wide slots, two per head for 15B); wider or odd heads are rejected at construction, loudly."""
    from esm_b200 import ESM2
    for L, E, H in [(1, 320, 20), (1, 480, 20), (1, 640, 20), (1, 1280, 20), (1, 256, 2)]:
        m = ESM2(num_layers=L, embed_dim=E, attention_heads=H)
        assert m.layers[0].self_attn.head_dim == E // H
    with pytest.raises(ValueError):
        ESM2(num_layers=1, embed_dim=512, attention_heads=2)   # head_dim 256
    with pytest.raises(ValueError):
        ESM2(num_layers=1, embed_dim=66, attention_heads=2)    # head_dim 33


def test_state_dict_keys_match_reference_layout():
    """keys/shapes the reference's checkpoints carry (SURVEY §7 data-layout notes; esm2.py:40-75)."""
    from esm_b200 import ESM2
    from oracle.weights import make_state_dict
    model = ESM2(num_layers=2, embed_dim=128, attention_heads=2)
    sd = make_state_dict(2, 128, 2)
    assert set(model.state_dict().keys()) == set(sd.keys())
    model.load_state_dict(sd, strict=True)
    assert model.lm_head.weight is model.embed_tokens.weight


def test_hot_kernels_run_on_the_tensor_cores():
    """The shipped library's GEMMs are wgmma kernels (HGMMA in the SASS) and its attention kernels use the warp-level
    tensor-core MMA (HMMA): no hot-path kernel computes its products on the FMA pipe."""
    import shutil
    import subprocess
    from esm_b200 import _lib
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump) or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("cuobjdump or the built library is not available")
    sass = subprocess.run([cuobjdump, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    counts, cur = {}, None
    for line in sass.splitlines():
        if "Function :" in line:
            cur = line.split("Function :")[1].strip()
            counts[cur] = {"HGMMA": 0, "HMMA": 0}
        elif cur:
            if "HGMMA" in line:
                counts[cur]["HGMMA"] += 1
            elif "HMMA" in line:
                counts[cur]["HMMA"] += 1
    gemms = [c for n, c in counts.items() if "gemm2_f16_kernel" in n]
    attn = [c for n, c in counts.items() if any(k in n for k in ("attention_fwd_kernel", "attention_probs", "tied_scores",
                                                                  "tied_pv"))]
    assert len(gemms) == 10 and all(c["HGMMA"] > 0 for c in gemms), gemms
    assert len(attn) >= 8 and all(c["HMMA"] > 0 for c in attn), attn
