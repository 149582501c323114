"""GPU (-m gpu): the UNMODIFIED reference running on top of libesmb200.so (INTEGRATION.md Option B, VERDICT r1 missing #3).

The reference package is imported from `oracle/_ref`, which build() makes by the recipe in oracle/reference.py
(git-ignored; it travels with the tree to the GPU machine).  `esm_b200.integration.patch_reference()` substitutes `esm.modules.TransformerLayer.forward`, the seam SURVEY
§8b names (`esm/modules.py:120-142` called from `esm/model/esm2.py:111-116`), exactly like the reference's own apex
FusedLayerNorm substitution (`esm/modules.py:68-81`); everything else — `ESM2.forward`'s loop, embedding prologue, LM
head, contact head — is the reference's own code executing on the GPU.
"""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def rel_fro(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


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


def _reference_model(esm, L, E, H, seed=0):
    from oracle.weights import make_state_dict
    sd = make_state_dict(L, E, H, seed=seed)
    model = esm.model.esm2.ESM2(num_layers=L, embed_dim=E, attention_heads=H, alphabet="ESM-1b")
    model.load_state_dict(sd, strict=True)
    return model.eval()


@pytest.mark.parametrize("name", ["tiny_L2_E128_H2", "mid_L3_E256_H4", "t6_8M_like_L6_E320_H20",
                                  "t48_15B_like_L2_E256_H2"])
def test_reference_esm2_forward_on_the_library(esm_ref, name, golden_dir):
    from esm_b200 import _lib, integration
    fx = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    cfg = fx["config"]
    model = _reference_model(esm_ref, cfg["num_layers"], cfg["embed_dim"], cfg["attention_heads"], cfg["seed"]).cuda()
    integration.patch_reference(esm_ref.modules)
    try:
        n0 = _lib.load().esmb200_launch_count()
        with torch.no_grad():
            out = model(fx["tokens"].cuda(), repr_layers=fx["repr_layers"], need_head_weights=True, return_contacts=True)
        torch.cuda.synchronize()
        launched = _lib.load().esmb200_launch_count() - n0
    finally:
        integration.unpatch_reference(esm_ref.modules)
    assert launched >= 7 * cfg["num_layers"], "the reference's layers did not go through libesmb200.so"
    for k, ref in fx["representations"].items():
        assert rel_fro(out["representations"][k].cpu(), ref) <= 3e-3, k
    assert rel_fro(out["logits"].cpu(), fx["logits"]) <= 4e-3
    L, H = cfg["num_layers"], cfg["attention_heads"]
    sub = out["attentions"][:, [0, L - 1]][:, :, [0, H - 1]].cpu()
    assert float((sub - fx["attentions_sub"]).abs().max()) <= 1e-2
    assert float((out["contacts"].cpu() - fx["contacts"]).abs().max()) <= 1e-2


def test_patched_reference_equals_reference_eager_on_the_same_gpu(esm_ref):
    """What `esm-extract` users run today (scripts/extract.py:70-72: model.cuda(), eager fp32) against the same model
    with the substituted layer, on the same device and tokens; plus ESMFold's fp16 variant (esmfold.py:59-62)."""
    from esm_b200 import integration
    from oracle.weights import make_tokens
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    L, E, H = 4, 640, 10
    model = _reference_model(esm_ref, L, E, H).cuda()
    tokens = make_tokens([200, 131], 202, seed=2, n_mask=1).cuda()
    with torch.no_grad():
        eager = model(tokens, repr_layers=[L])["representations"][L]
    integration.patch_reference(esm_ref.modules)
    try:
        with torch.no_grad():
            fast = model(tokens, repr_layers=[L])["representations"][L]
            fast16 = model.half()(tokens, repr_layers=range(L + 1))["representations"]
    finally:
        integration.unpatch_reference(esm_ref.modules)
    keep = tokens.ne(1)
    assert rel_fro(fast[keep], eager[keep]) <= 3e-3
    assert fast16[L].dtype == torch.float16 and sorted(fast16.keys()) == list(range(L + 1))
    assert rel_fro(fast16[L].float()[keep], eager[keep]) <= 8e-3  # fp16 weights + fp16 reference prologue/tail


def test_reference_650M_full_size_eager_vs_library(esm_ref):
    """BASELINE.json configs[1] at full size with the REAL reference on both sides: the unmodified `ESM2` of fair-esm
    (33 x 1280 x 20 heads) on the GPU in eager fp32 (TF32 off) against the same object with its TransformerLayer.forward
    substituted, T = 1024, two sequences (one padded to 700 residues): last representation, logits, contacts."""
    from esm_b200 import integration
    from oracle.weights import make_tokens
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    L, E, H = 33, 1280, 20
    model = _reference_model(esm_ref, L, E, H).cuda()
    tokens = make_tokens([1022, 700], 1024, seed=4, n_mask=3).cuda()
    with torch.no_grad():
        eager = model(tokens, repr_layers=[L], return_contacts=True)
        eager = {"rep": eager["representations"][L], "logits": eager["logits"], "contacts": eager["contacts"]}
    integration.patch_reference(esm_ref.modules)
    try:
        with torch.no_grad():
            fast = model(tokens, repr_layers=[L], return_contacts=True)
    finally:
        integration.unpatch_reference(esm_ref.modules)
    keep = tokens.ne(1)
    r = rel_fro(fast["representations"][L][keep], eager["rep"][keep])
    rl = rel_fro(fast["logits"][keep], eager["logits"][keep])
    rc = float((fast["contacts"] - eager["contacts"])[0].abs().max())  # sequence 0 has no padding
    print(f"PARITY reference_eager_650M_T1024 repr={r:.3e} logits={rl:.3e} contacts_abs={rc:.3e}", flush=True)
    assert r <= 3e-3 and rl <= 4e-3 and rc <= 1e-2


def test_cpu_tensors_keep_the_reference_path(esm_ref):
    """Like the FusedLayerNorm precedent: on CPU the substituted class runs the reference's own PyTorch code."""
    from esm_b200 import integration
    model = _reference_model(esm_ref, 1, 128, 2)
    tokens = torch.tensor([[0, 5, 6, 7, 8, 2]])
    with torch.no_grad():
        want = model(tokens, repr_layers=[1])["representations"][1]
    integration.patch_reference(esm_ref.modules)
    try:
        with torch.no_grad():
            got = model(tokens, repr_layers=[1])["representations"][1]
    finally:
        integration.unpatch_reference(esm_ref.modules)
    assert torch.equal(got, want)
