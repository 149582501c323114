"""GPU (-m gpu): contacts without the attention stack (esmb200_stack_contacts, ProteinLanguageModel.predict_contacts).

The contacts-only path must be bit-identical to forward(tokens, return_contacts=True)["contacts"] wherever the latter
runs, so every comparison below is torch.equal:

  * accumulator level: acc, row_part, col_part and the residual stream of the store-free fused pass
    (attention_probs_contact_kernel<DS, false>) against the storing pass, both DS, T from 1 to 4097, with and without
    padding and <eos>, head_dim 16 / 64 / 96 / 128, up to 40 heads; partials start as NaN so an unwritten one fails;
  * model level: predict_contacts against forward on the ESM-2 and ESM-1b goldens in every allowed precision,
    resident and after cpu_offload(), and after model.half(); the internal forward's representations too;
  * a 2049-token protein against the CPU oracle; peak device memory against the stack; extract_cli's files;
  * the entry point's refusals.
"""
import argparse
import ctypes
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)  # esm1b_weights

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CONTACT_ABS = 1e-2  # DESIGN.md section 4, contacts against the reference / oracle
EINVAL, EWORKSPACE = -1, -4


def esm2(L, E, H, seed=0):
    from esm_b200 import ESM2
    from oracle.weights import make_state_dict
    m = ESM2(num_layers=L, embed_dim=E, attention_heads=H)
    m.load_state_dict(make_state_dict(L, E, H, seed=seed), strict=True)
    return m.eval()


def esm1b(fx):
    from esm_b200 import ProteinBertModel
    from esm1b_weights import make_esm1b_state_dict
    cfg = fx["config"]
    args = argparse.Namespace(**cfg["model_args"])
    m = ProteinBertModel(args, "roberta_large")
    m.load_state_dict(make_esm1b_state_dict(cfg["num_layers"], cfg["embed_dim"], cfg["attention_heads"],
                                            seed=cfg["seed"], emb_layer_norm_before=args.emb_layer_norm_before),
                      strict=True)
    return m.eval()


# ---- accumulator level ------------------------------------------------------------------------------------------
def _job(model, B, T, lo, hi, keep):
    from esm_b200 import _lib
    L, H = model.num_layers, model.attention_heads
    nt, S = (T + 127) // 128, hi - lo
    st = {"keep": keep, "acc": torch.zeros((B, S, S), device=DEV),
          "row": torch.full((L, B, H, 4 * nt, S), float("nan"), device=DEV),
          "col": torch.full((L, B, H, 4 * nt, S), float("nan"), device=DEV),
          "w": torch.randn((L, H), generator=torch.Generator().manual_seed(T)).to(DEV)}
    job = _lib.ContactJob()
    job.weights, job.keep = st["w"].data_ptr(), keep.data_ptr() if keep is not None else None
    job.acc, job.row_part, job.col_part = st["acc"].data_ptr(), st["row"].data_ptr(), st["col"].data_ptr()
    job.lo, job.hi = lo, hi
    st["job"] = job
    return st


def storing_and_store_free(model, tokens, lo, hi, keep):
    """run_stack with the storing fused pass (the forward's) and with the store-free one, same inputs"""
    from esm_b200.model import run_stack
    B, T = tokens.shape
    L, E = model.num_layers, model.embed_dim
    out = []
    with torch.no_grad(), torch.cuda.device(DEV):
        x0 = torch.empty((B, T, E), device=DEV)
        model._embed(tokens, x0)
        cos, sin = model._rope_tables(T)
        mask = tokens.eq(model.padding_idx)
        for contacts_only in (False, True):
            x = x0.clone()
            st = _job(model, B, T, lo, hi, keep)
            run_stack(list(model.layers), x, mask, cos, sin, None, [] if contacts_only else list(range(L)),
                      zero_pad_rows=True, contact_job=st["job"], contacts_only=contacts_only)
            out.append((x, st))
    torch.cuda.synchronize()
    return out


# (L, E, H, T, residue lengths or None = no <cls>/<eos>/padding): crop [lo, hi) = [1, T-1) with <eos> masking when
# lengths are given, else [0, T) without keep
ACC_CASES = [
    (2, 128, 2, 1, None),                 # one position
    (2, 128, 2, 2, None),
    (2, 320, 20, 127, [125, 60]),         # head_dim 16 in 64-wide slots, padded second sequence
    (2, 128, 2, 128, [126, 126]),         # one full tile, no padding
    (2, 256, 2, 129, [127, 100]),         # DS = 2 (head_dim 128), one column past the tile
    (1, 2560, 40, 1000, [998, 517, 90]),  # 40 heads of 64 (3B width); later key tiles of two sequences not live
    (2, 192, 2, 1027, [1025, 300]),       # DS = 2 with head_dim 96
    (1, 5120, 40, 300, [298, 171]),       # 40 heads of 128 (15B width)
    (1, 256, 2, 4097, [4095, 2000]),      # 33 tiles, DS = 2
    (1, 128, 2, 4097, None),              # 33 tiles, DS = 1, no crop, no padding
]


@pytest.mark.parametrize("L,E,H,T,lengths", ACC_CASES)
def test_store_free_pass_equals_storing_pass(L, E, H, T, lengths):
    from oracle.weights import make_tokens
    model = esm2(L, E, H, seed=T).to(DEV)
    if lengths is None:
        tokens = torch.randint(4, 24, (2, T), generator=torch.Generator().manual_seed(T)).to(DEV)
        lo, hi, keep = 0, T, None
    else:
        tokens = make_tokens(lengths, T, seed=T, n_mask=1).to(DEV)
        lo, hi, keep = 1, T - 1, tokens.ne(model.eos_idx).to(torch.uint8).contiguous()
    (xa, a), (xb, b) = storing_and_store_free(model, tokens, lo, hi, keep)
    for name in ("row", "col"):
        assert not bool(b[name].isnan().any()), f"store-free pass left a {name} partial unwritten"
        assert torch.equal(a[name], b[name]), name
    assert torch.equal(a["acc"], b["acc"])
    assert torch.equal(xa, xb)
    assert float(b["acc"].abs().max()) > 0


# ---- model level ------------------------------------------------------------------------------------------------
def _check_model(model, tokens, repr_layers):
    """predict_contacts and the internal forward against forward(return_contacts=True), bit for bit"""
    ref = model(tokens, repr_layers=repr_layers, return_contacts=True)
    got = model._contacts_forward(tokens, repr_layers=repr_layers)
    assert set(got) == {"representations", "contacts"}
    assert got["contacts"].dtype == ref["contacts"].dtype
    assert torch.equal(got["contacts"], ref["contacts"])
    assert got["representations"].keys() == ref["representations"].keys()
    for k, v in ref["representations"].items():
        assert torch.equal(got["representations"][k], v), k
    assert torch.equal(model.predict_contacts(tokens), ref["contacts"])


ESM2_GOLDENS = ["t6_8M_like_L6_E320_H20", "mid_L3_E256_H4", "t48_15B_like_L2_E256_H2"]
ESM1B_GOLDENS = ["esm1b_tiny_L2_E128_H2", "esm1b_mid_L3_E256_H4", "esm1b_edge_L1_E128_H2_T1024"]
MODES = [("fp16", False), ("fp8", False), ("fp32x3", False), ("fp16", True), ("fp32x3", True)]


def _allowed(model, precision):
    return precision != "fp32x3" or model.embed_dim // model.attention_heads <= 64


@pytest.mark.parametrize("precision,offload", MODES)
@pytest.mark.parametrize("name", ESM2_GOLDENS + ESM1B_GOLDENS)
def test_predict_contacts_equals_forward_on_goldens(name, precision, offload, golden_dir):
    fx = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    if name.startswith("esm1b"):
        model = esm1b(fx)
    else:
        cfg = fx["config"]
        model = esm2(cfg["num_layers"], cfg["embed_dim"], cfg["attention_heads"], cfg["seed"])
    if not _allowed(model, precision):
        with pytest.raises(ValueError):
            model.set_precision(precision)
        return
    model.set_precision(precision)
    model = model.cpu_offload(DEV) if offload else model.to(DEV)
    assert all(layer.offloaded == offload for layer in model.layers)
    _check_model(model, fx["tokens"].to(DEV), list(range(model.num_layers + 1)))


@pytest.mark.parametrize("precision", ["fp16", "fp8", "fp32x3"])
@pytest.mark.parametrize("name", ["mid_L3_E256_H4", "esm1b_tiny_L2_E128_H2"])
def test_predict_contacts_after_half(name, precision, golden_dir):
    fx = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    if name.startswith("esm1b"):
        model = esm1b(fx)
    else:
        cfg = fx["config"]
        model = esm2(cfg["num_layers"], cfg["embed_dim"], cfg["attention_heads"], cfg["seed"])
    model = model.set_precision(precision).to(DEV).half()
    tokens = fx["tokens"].to(DEV)
    assert model.predict_contacts(tokens).dtype == torch.float16
    _check_model(model, tokens, [0, model.num_layers])


def test_long_protein_against_oracle():
    """T = 2049: past the fp32x3 contact limit and past ESM-1b's positions; the fp16 path against the CPU oracle"""
    from oracle import esm2_oracle
    from oracle.weights import make_state_dict, make_tokens
    L, E, H = 2, 128, 2
    sd = make_state_dict(L, E, H, seed=11)
    model = esm2(L, E, H, seed=11).to(DEV)
    tokens = make_tokens([2047, 1500], 2049, seed=11, n_mask=2)
    got = model.predict_contacts(tokens.to(DEV))
    ref = esm2_oracle.esm2_forward(sd, L, H, tokens, return_contacts=True)["contacts"]
    err = float((got.cpu() - ref).abs().max())
    print(f"PARITY contacts_only T2049 max_abs={err:.3e}")
    assert got.shape == ref.shape and err <= CONTACT_ABS
    assert torch.equal(got, model(tokens.to(DEV), return_contacts=True)["contacts"])


# ---- memory -----------------------------------------------------------------------------------------------------
def test_peak_memory_is_the_partials_not_the_stack():
    """650M width, 6 layers, 8 x 1024: the stack is 4 GB; predict_contacts holds the partials (1/16 of it), the
    accumulator and output [B,S,S], the residual stream and the (cached) workspace, plus 16 MB of small tensors."""
    from esm_b200 import _lib
    from oracle.weights import make_tokens
    L, E, H, B, T = 6, 1280, 20, 8, 1024
    model = esm2(L, E, H).to(DEV)
    tokens = make_tokens([1022] * 6 + [700, 300], T, seed=5).to(DEV)
    S = T - 2
    lib = _lib.load()
    row, col, scratch = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(lib.esmb200_stack_contacts_bytes(L, H, B, T, S, 0, ctypes.byref(row), ctypes.byref(col),
                                                ctypes.byref(scratch)))
    stack = 4 * B * L * H * T * T
    ws = lib.esmb200_workspace_bytes(E, H, 4 * E, B, T, 0)
    bound = row.value + col.value + 2 * 4 * B * S * S + 4 * B * T * E + ws + (16 << 20)

    def peak(fn):
        fn()  # warm-up: the workspace is cached per stream
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(DEV)
        torch.cuda.reset_peak_memory_stats(DEV)
        out = fn()
        torch.cuda.synchronize()
        p = torch.cuda.max_memory_allocated(DEV) - base
        del out
        return p

    p_contacts = peak(lambda: model.predict_contacts(tokens))
    p_forward = peak(lambda: model(tokens, return_contacts=True)["contacts"])
    print(f"MEMORY stack={stack / 1e9:.3f} GB partials={(row.value + col.value) / 1e9:.3f} GB "
          f"bound={bound / 1e9:.3f} GB predict_contacts={p_contacts / 1e9:.3f} GB forward={p_forward / 1e9:.3f} GB")
    assert scratch.value == 0
    assert p_contacts <= bound
    assert p_contacts < stack / 8
    assert p_forward > stack


# ---- extract_cli ------------------------------------------------------------------------------------------------
def test_extract_cli_contacts_equal_forward(tmp_path):
    """every file's contacts and representations equal the forward's on the batch extract_cli formed, bit for bit"""
    from esm_b200 import extract_cli, pretrained
    from esm_b200.data import FastaBatchedDataset
    from esm_b200.extract import mean_pool
    from oracle.weights import make_state_dict
    L, E, H = 2, 128, 2
    sd = make_state_dict(L, E, H, seed=4)
    ckpt = tmp_path / "esm2_tiny.pt"
    torch.save({"cfg": {"model": {"encoder_layers": L, "encoder_embed_dim": E, "encoder_attention_heads": H,
                                  "token_dropout": True}},
                "model": {("encoder.sentence_encoder." + k): v for k, v in sd.items()}}, ckpt)
    g = torch.Generator().manual_seed(4)
    aa = "ACDEFGHIKLMNPQRSTVWY"
    seqs = {f"p{i}": "".join(aa[j] for j in torch.randint(0, 20, (n,), generator=g).tolist())
            for i, n in enumerate([300, 27, 181, 3, 250, 96])}
    fasta = tmp_path / "in.fasta"
    fasta.write_text("".join(f">{k}\n{v}\n" for k, v in seqs.items()))
    outdir = tmp_path / "out"
    args = argparse.Namespace(model_location=str(ckpt), fasta_file=fasta, output_dir=outdir, toks_per_batch=700,
                              repr_layers=[0, -1], include=["mean", "per_tok", "bos", "contacts"],
                              truncation_seq_length=1022)
    assert extract_cli.run(args) == len(seqs)
    model, alphabet = pretrained.load_model_and_alphabet(str(ckpt))
    model = model.eval().to(DEV)
    dataset = FastaBatchedDataset.from_file(fasta)
    to_tokens = alphabet.get_batch_converter(1022)
    seen = 0
    for idxs in dataset.get_batch_indices(700, extra_toks_per_seq=1):
        labels, strs, toks = to_tokens([dataset[i] for i in idxs])
        out = model(toks.to(DEV), repr_layers=[0, L], return_contacts=True)
        lengths = torch.tensor([len(s) for s in strs], dtype=torch.int32, device=DEV)
        for i, label in enumerate(labels):
            n = len(strs[i])
            r = torch.load(outdir / f"{label}.pt", weights_only=False)
            assert torch.equal(r["contacts"], out["contacts"][i, :n, :n].cpu())
            for layer in (0, L):
                t = out["representations"][layer]
                assert torch.equal(r["representations"][layer], t[i, 1:n + 1].cpu())
                assert torch.equal(r["bos_representations"][layer], t[i, 0].cpu())
                assert torch.equal(r["mean_representations"][layer], mean_pool(t, lengths)[i].cpu())
            seen += 1
    assert seen == len(seqs)


# ---- refusals of the entry point ----------------------------------------------------------------------------------
def _call(layers, x, B, T, job, scratch=None, scratch_bytes=0, ws=None, ws_bytes=None, ring=None, ring_bytes=0,
          copy=None, repr_out=None):
    from esm_b200 import _lib
    from esm_b200.model import _stream
    lib = _lib.load()
    n = len(layers)
    handles = (ctypes.c_void_p * n)(*[l.handle() for l in layers])
    first = layers[0]
    if ws is None:
        nbytes = lib.esmb200_workspace_bytes(first.embed_dim, first.attention_heads, first.ffn_embed_dim, B, T,
                                             first.precision)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    rc = lib.esmb200_stack_contacts(handles, n, x.data_ptr(), None, B, T, None, None, repr_out,
                                    ctypes.byref(job) if job is not None else None,
                                    scratch.data_ptr() if scratch is not None else None, scratch_bytes,
                                    ws.data_ptr(), ws.numel() if ws_bytes is None else ws_bytes,
                                    ring.data_ptr() if ring is not None else None, ring_bytes,
                                    ctypes.c_void_p(copy.cuda_stream) if copy is not None else None, _stream())
    return rc, lib.esmb200_last_error().decode()


def test_entry_point_refusals():
    from esm_b200 import _lib
    from esm_b200.model import _stream
    from oracle.weights import make_tokens
    lib = _lib.load()
    L, E, H = 2, 128, 2
    B, T = 2, 40
    fp16 = esm2(L, E, H).to(DEV)
    split = esm2(L, E, H).set_precision("fp32x3").to(DEV)
    tokens = make_tokens([38, 20], T).to(DEV)
    x = torch.zeros((B, T, E), device=DEV)
    st16 = fp16.contact_head.begin_contacts(tokens, L, H, 0)
    st3 = split.contact_head.begin_contacts(tokens, L, H, 1)
    for layer in list(fp16.layers) + list(split.layers):
        layer.handle()  # the packing launches kernels; what follows must not
    torch.cuda.synchronize()
    launches = lib.esmb200_launch_count()

    assert _call(list(fp16.layers), x, B, T, None)[0] == EINVAL  # null job
    rc, msg = _call(list(fp16.layers), x, B, T, st16["job"], ws_bytes=1024)
    assert rc == EWORKSPACE and "workspace" in msg
    rc, msg = _call(list(split.layers), x, B, T, st3["job"])  # no scratch
    assert rc == EWORKSPACE and "scratch" in msg
    scratch = st3["scratch"]
    rc, msg = _call(list(split.layers), x, B, T, st3["job"], scratch, scratch.nbytes - 4)
    assert rc == EWORKSPACE and "scratch" in msg
    rc, msg = _call([fp16.layers[0], split.layers[1]], x, B, T, st16["job"])  # mixed precision
    assert rc == EINVAL and "precision" in msg
    bad = _lib.ContactJob.from_buffer_copy(st16["job"])
    bad.hi = T + 1
    assert _call(list(fp16.layers), x, B, T, bad)[0] == EINVAL
    assert lib.esmb200_launch_count() == launches, "a refused call launched a kernel"

    # fp32x3 keeps esmb200_contact_accumulate's 1024-position limit, refused before any launch
    Tl = 1027
    tl = make_tokens([1025], Tl).to(DEV)
    xl = torch.zeros((1, Tl, E), device=DEV)
    stl = split.contact_head.begin_contacts(tl, L, H, 1)
    rc, msg = _call(list(split.layers), xl, 1, Tl, stl["job"], stl["scratch"], stl["scratch"].nbytes)
    assert rc == EINVAL and msg == "contact head supports at most 1024 positions"
    assert lib.esmb200_launch_count() == launches
    with pytest.raises(_lib.Esmb200Error, match="at most 1024 positions"):
        split.predict_contacts(tl)

    # resident and offloaded layers mixed
    off = esm2(L, E, H).cpu_offload(DEV)
    rc, msg = _call([fp16.layers[0], off.layers[1]], x, B, T, st16["job"])
    assert rc == EINVAL and "offloaded" in msg

    # esmb200_stack_forward keeps its contract: a contact job without attn_out is refused
    handles = (ctypes.c_void_p * L)(*[l.handle() for l in fp16.layers])
    ws = torch.empty(lib.esmb200_workspace_bytes(E, H, 4 * E, B, T, 0), dtype=torch.uint8, device=DEV)
    rc = lib.esmb200_stack_forward(handles, L, x.data_ptr(), None, B, T, None, None, None, None, 0, 1,
                                   ctypes.byref(st16["job"]), ws.data_ptr(), ws.numel(), _stream())
    assert rc == EINVAL and "attn_out" in lib.esmb200_last_error().decode()
