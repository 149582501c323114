"""esm_b200 — H100-native (sm_90a) ESM-2 transformer-layer forward behind the reference's Python API.

    from esm_b200 import pretrained
    model, alphabet = pretrained.esm2_t33_650M_UR50D()      # same call as esm.pretrained.*
    out = model.cuda()(tokens.cuda(), repr_layers=[33])      # same forward contract as esm.model.esm2.ESM2

    msa_model, msa_alphabet = pretrained.esm_msa1b_t12_100M_UR50S()   # MSA Transformer: tokens [B, R, C]
    esm1v_model, _ = pretrained.esm1v_t33_650M_UR90S_1()              # ESM-1b / ESM-1v: ProteinBertModel
    lp = variants.masked_marginals(esm1v_model.cuda(), tokens)          # variant scoring (predict.py), batched

Compute goes through the C ABI of libesmb200.so (include/esmb200.h); see DESIGN.md / INTEGRATION.md.
"""
from .alphabet import Alphabet, BatchConverter  # noqa: F401
from .model import ESM2, TransformerLayer  # noqa: F401
from .esm1 import ProteinBertModel  # noqa: F401
from .msa import AxialTransformerLayer, MSATransformer  # noqa: F401
from . import pretrained, variants  # noqa: F401

__version__ = "0.1.0"
