"""Model factories with the reference's names and return convention (/root/reference/esm/pretrained.py:24-28,
164-183, 344-397): each returns `(model, alphabet)`.

Weights: the reference downloads `https://dl.fbaipublicfiles.com/fair-esm/models/{name}.pt` (pretrained.py:53).
Here a checkpoint is loaded when it is found locally (torch hub cache or an explicit path, same file format and
key-upgrade rule as pretrained.py:164-183).  When it is not — there is no network in this environment — the factories
RAISE like the reference does when weights cannot be obtained; `allow_random_init=True` (benchmarks and tests) returns a
seeded random-init model instead, with a warning and `model.random_init = True`.
Loading is strict like pretrained.py:200-219: only `contact_head.regression.*` may be missing (with a warning).
The 15B model (head_dim 128) runs with two 64-wide column slots per head (DESIGN.md section 1).
"""
from __future__ import annotations

import os
import re
import warnings
from typing import Optional, Tuple

import torch

from argparse import Namespace

from .alphabet import Alphabet
from .model import ESM2

# name -> (num_layers, embed_dim, attention_heads)   (README.md:477-482 + checkpoint cfg, SURVEY §8)
ESM2_ARCH = {
    "esm2_t6_8M_UR50D": (6, 320, 20),
    "esm2_t12_35M_UR50D": (12, 480, 20),
    "esm2_t30_150M_UR50D": (30, 640, 20),
    "esm2_t33_650M_UR50D": (33, 1280, 20),
    "esm2_t36_3B_UR50D": (36, 2560, 40),
    "esm2_t48_15B_UR50D": (48, 5120, 40),
}


def _hub_path(name: str) -> str:
    return os.path.join(torch.hub.get_dir(), "checkpoints", f"{name}.pt")


def _upgrade_state_dict(state_dict):
    """pretrained.py:164-170: strip the fairseq prefixes."""
    prefixes = ["encoder.sentence_encoder.", "encoder."]
    pattern = re.compile("^" + "|".join(prefixes))
    return {pattern.sub("", k): v for k, v in state_dict.items()}


def _load_checked(model, state_dict, what: str) -> None:
    """pretrained.py:200-219: every key must match, except that a checkpoint without its `-contact-regression.pt`
    companion may lack `contact_head.regression.*` (warned, as the reference does)."""
    expected = set(model.state_dict().keys())
    found = set(state_dict.keys())
    missing = expected - found
    unexpected = found - expected
    regression = {"contact_head.regression.weight", "contact_head.regression.bias"}
    errors = []
    if missing - regression:
        errors.append(f"Missing key(s) in state_dict: {sorted(missing - regression)}.")
    if unexpected:
        errors.append(f"Unexpected key(s) in state_dict: {sorted(unexpected)}.")
    if errors:
        raise RuntimeError("Error(s) in loading state_dict for {}:\n\t{}".format(what, "\n\t".join(errors)))
    if missing:
        warnings.warn("Regression weights not found, predicting contacts will not produce correct results.")
    model.load_state_dict(state_dict, strict=not missing)


def _random_init_or_raise(model_name: str, path: str, allow_random_init: bool) -> None:
    allow = allow_random_init or os.environ.get("ESMB200_ALLOW_RANDOM_INIT", "") == "1"
    if not allow:
        raise FileNotFoundError(
            f"{model_name}: no checkpoint at {path} and no network to download it (pretrained.py:53). Pass a local "
            f".pt path, place the file in the torch hub cache, or ask for seeded random weights explicitly with "
            f"allow_random_init=True (benchmarks / tests only).")
    warnings.warn(f"{model_name}: checkpoint {path} not found — returning a seeded RANDOM-INIT model "
                  f"(model.random_init = True); its outputs are meaningless as embeddings.")


def load_model_and_alphabet_local(model_location: str):
    """pretrained.py:67-77 / 164-183 for ESM-2: reads {"cfg": {"model": ...}, "model": sd}.  A v1 checkpoint
    ({"args": Namespace, "model": sd}: ESM-1b / ESM-1v) is read by the v1 `roberta_large` loader (pretrained.py:85-101)."""
    data = torch.load(str(model_location), map_location="cpu", weights_only=False)
    if "cfg" not in data and "args" in data:
        return _load_esm1b(model_location, data)
    cfg = data["cfg"]["model"]
    get = (lambda k: cfg[k]) if isinstance(cfg, dict) else (lambda k: getattr(cfg, k))
    model = ESM2(num_layers=get("encoder_layers"), embed_dim=get("encoder_embed_dim"),
                 attention_heads=get("encoder_attention_heads"), alphabet="ESM-1b",
                 token_dropout=get("token_dropout"))
    sd = _upgrade_state_dict(data["model"])
    reg = str(model_location)[:-3] + "-contact-regression.pt"
    if os.path.exists(reg):
        sd.update(torch.load(reg, map_location="cpu", weights_only=False)["model"])
    _load_checked(model, sd, "ESM2")
    model.random_init = False
    return model.eval(), model.alphabet


def load_model_and_alphabet(model_name: str, seed: int = 0, allow_random_init: bool = False,
                            device=None) -> Tuple[ESM2, Alphabet]:
    """`device`: where a random-init model is created (e.g. "cuda": a 3B-parameter init takes seconds there, a minute
    on the CPU); checkpoints are loaded on the CPU like the reference does."""
    if model_name.endswith(".pt"):
        return load_model_and_alphabet_local(model_name)
    if model_name in ESM1B_ARCH:
        return load_esm1b_model_and_alphabet(model_name, seed, allow_random_init, device)
    if model_name.startswith("esm1_"):
        raise ValueError(f"{model_name!r} is an ESM-1 model: ESM-1 (bias_kv attention) is not supported by esm_b200")
    if model_name not in ESM2_ARCH:
        raise ValueError(f"unknown model {model_name!r}: this loader covers ESM-2 and ESM-1b / ESM-1v (the MSA "
                         "Transformer loads through load_msa_model_and_alphabet)")
    path = _hub_path(model_name)
    if os.path.exists(path):
        return load_model_and_alphabet_local(path)
    _random_init_or_raise(model_name, path, allow_random_init)
    L, E, H = ESM2_ARCH[model_name]
    gen_state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    if device is not None:
        with torch.device(device):
            model = ESM2(num_layers=L, embed_dim=E, attention_heads=H, alphabet="ESM-1b")
    else:
        model = ESM2(num_layers=L, embed_dim=E, attention_heads=H, alphabet="ESM-1b")
    torch.random.set_rng_state(gen_state)
    model.random_init = True
    return model.eval(), model.alphabet


def esm2_t33_650M_UR50D(allow_random_init: bool = False):
    return load_model_and_alphabet("esm2_t33_650M_UR50D", allow_random_init=allow_random_init)


def esm2_t36_3B_UR50D(allow_random_init: bool = False):
    return load_model_and_alphabet("esm2_t36_3B_UR50D", allow_random_init=allow_random_init)


def esm2_t6_8M_UR50D(allow_random_init: bool = False):
    return load_model_and_alphabet("esm2_t6_8M_UR50D", allow_random_init=allow_random_init)


def esm2_t12_35M_UR50D(allow_random_init: bool = False):
    return load_model_and_alphabet("esm2_t12_35M_UR50D", allow_random_init=allow_random_init)


def esm2_t30_150M_UR50D(allow_random_init: bool = False):
    return load_model_and_alphabet("esm2_t30_150M_UR50D", allow_random_init=allow_random_init)


def esm2_t48_15B_UR50D(allow_random_init: bool = False):
    return load_model_and_alphabet("esm2_t48_15B_UR50D", allow_random_init=allow_random_init)


# ---- ESM-1b / ESM-1v: ProteinBertModel, arch "roberta_large" (pretrained.py:85-101, 267-341) ----------------------
_ESM1B_ARGS = dict(arch="roberta_large", layers=33, embed_dim=1280, ffn_embed_dim=5120, attention_heads=20,
                   max_positions=1024, emb_layer_norm_before=True, token_dropout=True)
ESM1B_ARCH = {  # name -> constructor arguments (the checkpoints' args after the prefix upgrade)
    "esm1b_t33_650M_UR50S": _ESM1B_ARGS,
    "esm1v_t33_650M_UR90S_1": _ESM1B_ARGS,
    "esm1v_t33_650M_UR90S_2": _ESM1B_ARGS,
    "esm1v_t33_650M_UR90S_3": _ESM1B_ARGS,
    "esm1v_t33_650M_UR90S_4": _ESM1B_ARGS,
    "esm1v_t33_650M_UR90S_5": _ESM1B_ARGS,
}


def _upgrade_esm1b_checkpoint(data, alphabet: Alphabet):
    """pretrained.py:90-100: strip "encoder_" from argument names and the "sentence_encoder." / "encoder." prefixes
    from parameter names, zero the <mask> row of embed_tokens (token dropout), and infer emb_layer_norm_before from
    the keys."""
    strip_arg = lambda k: "".join(k.split("encoder_")[1:] if "encoder" in k else k)
    strip1 = lambda k: "".join(k.split("encoder.")[1:] if "encoder" in k else k)
    strip2 = lambda k: "".join(k.split("sentence_encoder.")[1:] if "sentence_encoder" in k else k)
    args = {strip_arg(k): v for k, v in vars(data["args"]).items()}
    state = {strip1(strip2(k)): v for k, v in data["model"].items()}
    state["embed_tokens.weight"][alphabet.mask_idx].zero_()
    args["emb_layer_norm_before"] = any(k.startswith("emb_layer_norm_before") for k in state)
    return args, state


def _load_esm1b(model_location: str, data):
    from .esm1 import ProteinBertModel
    arch = getattr(data["args"], "arch", None)
    if arch == "protein_bert_base":
        raise ValueError(f"{model_location}: an ESM-1 checkpoint; ESM-1 (bias_kv attention) is not supported by esm_b200")
    if arch != "roberta_large":
        raise ValueError(f"{model_location}: unsupported v1 checkpoint architecture {arch!r}")
    reg = str(model_location)[:-3] + "-contact-regression.pt"
    if os.path.exists(reg):  # ESM-1b ships one; ESM-1v has none (pretrained.py:18-21), which warns below
        data["model"].update(torch.load(reg, map_location="cpu", weights_only=False)["model"])
    alphabet = Alphabet.from_architecture("roberta_large")
    args, state = _upgrade_esm1b_checkpoint(data, alphabet)
    model = ProteinBertModel(Namespace(**args), alphabet)
    _load_checked(model, state, "ProteinBertModel")
    model.random_init = False
    return model.eval(), alphabet


def load_esm1b_model_and_alphabet(model_name: str, seed: int = 0, allow_random_init: bool = False, device=None):
    """ESM-1b / ESM-1v by name (hub cache) or from a local v1 .pt file."""
    from .esm1 import ProteinBertModel
    if model_name.endswith(".pt"):
        return load_model_and_alphabet_local(model_name)
    if model_name not in ESM1B_ARCH:
        raise ValueError(f"unknown ESM-1b / ESM-1v model {model_name!r}")
    path = _hub_path(model_name)
    if os.path.exists(path):
        return load_model_and_alphabet_local(path)
    _random_init_or_raise(model_name, path, allow_random_init)
    gen_state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    alphabet = Alphabet.from_architecture("roberta_large")
    if device is not None:
        with torch.device(device):
            model = ProteinBertModel(Namespace(**ESM1B_ARCH[model_name]), alphabet)
    else:
        model = ProteinBertModel(Namespace(**ESM1B_ARCH[model_name]), alphabet)
    torch.random.set_rng_state(gen_state)
    model.random_init = True
    return model.eval(), alphabet


def esm1b_t33_650M_UR50S(allow_random_init: bool = False):
    return load_esm1b_model_and_alphabet("esm1b_t33_650M_UR50S", allow_random_init=allow_random_init)


def esm1v_t33_650M_UR90S(allow_random_init: bool = False):
    """Alias of esm1v_t33_650M_UR90S_1, like the reference (pretrained.py:285-291)."""
    return esm1v_t33_650M_UR90S_1(allow_random_init=allow_random_init)


def esm1v_t33_650M_UR90S_1(allow_random_init: bool = False):
    return load_esm1b_model_and_alphabet("esm1v_t33_650M_UR90S_1", allow_random_init=allow_random_init)


def esm1v_t33_650M_UR90S_2(allow_random_init: bool = False):
    return load_esm1b_model_and_alphabet("esm1v_t33_650M_UR90S_2", allow_random_init=allow_random_init)


def esm1v_t33_650M_UR90S_3(allow_random_init: bool = False):
    return load_esm1b_model_and_alphabet("esm1v_t33_650M_UR90S_3", allow_random_init=allow_random_init)


def esm1v_t33_650M_UR90S_4(allow_random_init: bool = False):
    return load_esm1b_model_and_alphabet("esm1v_t33_650M_UR90S_4", allow_random_init=allow_random_init)


def esm1v_t33_650M_UR90S_5(allow_random_init: bool = False):
    return load_esm1b_model_and_alphabet("esm1v_t33_650M_UR90S_5", allow_random_init=allow_random_init)


def _esm1_unsupported(name: str):
    def factory(*args, **kwargs):
        raise ValueError(f"{name!r} is an ESM-1 model: ESM-1 (bias_kv attention) is not supported by esm_b200")
    factory.__name__ = name
    return factory


esm1_t34_670M_UR50S = _esm1_unsupported("esm1_t34_670M_UR50S")
esm1_t34_670M_UR50D = _esm1_unsupported("esm1_t34_670M_UR50D")
esm1_t34_670M_UR100 = _esm1_unsupported("esm1_t34_670M_UR100")
esm1_t12_85M_UR50S = _esm1_unsupported("esm1_t12_85M_UR50S")
esm1_t6_43M_UR50S = _esm1_unsupported("esm1_t6_43M_UR50S")


# ---- MSA Transformer (pretrained.py:104-125, 293-300) -----------------------------------------------------------
MSA_ARCH = {  # name -> constructor arguments (the checkpoints' args)
    "esm_msa1_t12_100M_UR50S": dict(layers=12, embed_dim=768, ffn_embed_dim=3072, attention_heads=12,
                                    max_positions=1024, embed_positions_msa=True),
    "esm_msa1b_t12_100M_UR50S": dict(layers=12, embed_dim=768, ffn_embed_dim=3072, attention_heads=12,
                                     max_positions=1024, embed_positions_msa=True),
}


def _upgrade_msa_checkpoint(data):
    """pretrained.py:110-123: strip the fairseq "encoder." / "sentence_encoder." prefixes from argument and parameter
    names, swap "row" <-> "column" in parameter names (the checkpoints were trained with the two attention blocks
    named the other way round), and take the width of msa_position_embedding from the tensor (1 in the first release)."""
    strip_arg = lambda k: "".join(k.split("encoder_")[1:]) if "encoder" in k else k
    strip1 = lambda k: "".join(k.split("encoder.")[1:]) if "encoder" in k else k
    strip2 = lambda k: "".join(k.split("sentence_encoder.")[1:]) if "sentence_encoder" in k else k
    swap = lambda k: k.replace("row", "column") if "row" in k else k.replace("column", "row")
    args = {strip_arg(k): v for k, v in vars(data["args"]).items()}
    state = {strip1(strip2(swap(k))): v for k, v in data["model"].items()}
    if args.get("embed_positions_msa", False):
        args["embed_positions_msa_dim"] = state["msa_position_embedding"].size(-1)
    return args, state


def load_msa_model_and_alphabet_local(model_location: str):
    from .msa import MSATransformer
    data = torch.load(str(model_location), map_location="cpu", weights_only=False)
    reg = str(model_location)[:-3] + "-contact-regression.pt"
    has_reg = os.path.exists(reg)
    if has_reg:
        data["model"].update(torch.load(reg, map_location="cpu", weights_only=False)["model"])
    args, state = _upgrade_msa_checkpoint(data)
    alphabet = Alphabet.from_architecture("msa_transformer")
    model = MSATransformer(Namespace(**args), alphabet)
    _load_checked(model, state, "MSATransformer")
    model.random_init = False
    return model.eval(), alphabet


def load_msa_model_and_alphabet(model_name: str, seed: int = 0, allow_random_init: bool = False, device=None):
    from .msa import MSATransformer
    if model_name.endswith(".pt"):
        return load_msa_model_and_alphabet_local(model_name)
    if model_name not in MSA_ARCH:
        raise ValueError(f"unknown MSA Transformer model {model_name!r}")
    path = _hub_path(model_name)
    if os.path.exists(path):
        return load_msa_model_and_alphabet_local(path)
    _random_init_or_raise(model_name, path, allow_random_init)
    gen_state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    alphabet = Alphabet.from_architecture("msa_transformer")
    if device is not None:
        with torch.device(device):
            model = MSATransformer(Namespace(**MSA_ARCH[model_name]), alphabet)
    else:
        model = MSATransformer(Namespace(**MSA_ARCH[model_name]), alphabet)
    torch.random.set_rng_state(gen_state)
    model.random_init = True
    return model.eval(), alphabet


def esm_msa1_t12_100M_UR50S(allow_random_init: bool = False):
    return load_msa_model_and_alphabet("esm_msa1_t12_100M_UR50S", allow_random_init=allow_random_init)


def esm_msa1b_t12_100M_UR50S(allow_random_init: bool = False):
    return load_msa_model_and_alphabet("esm_msa1b_t12_100M_UR50S", allow_random_init=allow_random_init)
