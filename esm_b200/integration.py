"""INTEGRATION.md "Option B" as a runtime patch: run the UNMODIFIED reference's `ESM2.forward` with its
`TransformerLayer.forward` dispatched to libesmb200.so.

The reference has no plugin registry; its only precedent for swapping in native code is the import-time substitution
of apex's FusedLayerNorm (/root/reference/esm/modules.py:68-81).  `patch_reference()` does the same thing for the
transformer block at run time:

    import esm, esm_b200.integration
    esm_b200.integration.patch_reference()            # esm.modules.TransformerLayer.forward -> C ABI on CUDA tensors
    model, alphabet = esm.pretrained.esm2_t33_650M_UR50D()
    out = model.cuda()(tokens.cuda(), repr_layers=[33])   # the reference's own esm2.py:77-144 loop, H100 kernels inside

Layers on CUDA tensors without bias_k are dispatched — exactly the seam SURVEY §8b names (`esm/modules.py:120-142`
called from `esm/model/esm2.py:111-116` and `esm/model/esm1.py:155-158`): the rotary ESM-2 layers, and the ESM-1b /
ESM-1v layers of `ProteinBertModel` (learned positions, added by the reference's own prologue; the layer runs without
rotary tables).  ESM-1 layers (bias_kv attention) and CPU tensors keep the reference's PyTorch path, like the
FusedLayerNorm fallback.  This is the drop-in proof, not the fast path: the reference's loop still transposes to
(T,B,E) and round-trips through Python between layers, and its embedding prologue / LM head / contact head stay
PyTorch; `esm_b200.ESM2` and `esm_b200.ProteinBertModel` run the whole loop in one C call.
"""
from __future__ import annotations

from .model import LayerBinding, layer_forward

_ORIGINAL = {}


def _dispatchable(layer, x) -> bool:
    """CUDA input and no bias_k (ESM-1's extra learned key/value): a rotary ESM-2 layer, or an ESM-1b / ESM-1v layer
    that has neither rotary embedding nor bias_kv."""
    if not x.is_cuda or getattr(layer.self_attn, "bias_k", None) is not None:
        return False
    rotary = getattr(layer, "use_rotary_embeddings", False)
    return (getattr(layer.self_attn, "rot_emb", None) is not None) == bool(rotary)


def patch_reference(esm_modules=None) -> None:
    """Substitute `esm.modules.TransformerLayer.forward`.  `esm_modules`: the reference's `esm.modules` module (default:
    `import esm.modules`)."""
    if esm_modules is None:
        import esm.modules as esm_modules  # the reference package, wherever the caller's sys.path finds it
    cls = esm_modules.TransformerLayer
    if cls in _ORIGINAL:
        return
    original = cls.forward

    def forward(self, x, self_attn_mask=None, self_attn_padding_mask=None, need_head_weights=False):
        if self_attn_mask is not None or not _dispatchable(self, x):
            return original(self, x, self_attn_mask=self_attn_mask, self_attn_padding_mask=self_attn_padding_mask,
                            need_head_weights=need_head_weights)
        binding = self.__dict__.get("_esmb200_binding")
        if binding is None:
            binding = LayerBinding(self)
            self.__dict__["_esmb200_binding"] = binding  # plain attribute: not a parameter, buffer or submodule
        return layer_forward(binding, x, None, self_attn_padding_mask, need_head_weights)

    _ORIGINAL[cls] = original
    cls.forward = forward


def unpatch_reference(esm_modules=None) -> None:
    if esm_modules is None:
        import esm.modules as esm_modules
    cls = esm_modules.TransformerLayer
    if cls in _ORIGINAL:
        cls.forward = _ORIGINAL.pop(cls)
