"""GPU (-m gpu): the layer stacks against a layer-by-layer replay of the same kernels through the single-kernel C-ABI
entry points (tests/stack_replay.py), bit for bit, and every stage of the replay against float64 on its own inputs.

The replay packs the weights itself and takes the LayerNorm eps, the q scale and the rotary tables from the reference's
definitions, so a stack that uses a slightly wrong parameter (an eps, a q scale one fp32 ulp off, a table, a bias
pointer, a batch stride, a ring slot) gives other bits, however small the effect on the numbers.  The float64 stages then
hold each kernel to its error bound at the benchmark shapes, where a fixed model-level tolerance would let a small
systematic error through.

Cases (head_dim 64; random weights from oracle.weights, each stack cycling through a few distinct layers):
  * 650M width (E 1280, H 20), 33 layers, T = 1024, B = 3 ragged: fp16, fp32x3 and fp8 resident; fp16 and fp32x3
    after offloading (esmb200_stack_forward_streamed); fp16 with programmatic dependent launch;
  * 3B width (E 2560, H 40), 36 layers, T = 512: fp16 through esmb200_stack_contacts (its contact accumulators equal
    to the storing pass's, whose maps equal the replay's), and fp8;
  * ESM-1b (no rotary tables), 33 layers, T = 1024 ragged: fp16, fp32x3, fp8;
  * esmb200_stack_contacts in fp32x3 against a replay that folds each layer's maps with esmb200_contact_accumulate;
  * ESM2.forward: the logits and the post-LN last representation against a replay of the LM-head chain, each of its
    stages against float64;
  * MSA-1b (E 768, H 12), 12 layers: run_axial_stack against AxialTransformerLayer.forward_batch_major(need_probs=True)
    and the replay, layer after layer, at 2 x 32 x 256 padded, depths R = 6 and 17 (where fp32(0.125 / sqrt(R)) differs
    from the reference's fp32(64 ** -0.5 / sqrt(R))), fp16 and fp32x3, with every stage against float64 (the column
    maps at every query row of every live column), and 128 x 512 in fp16;
  * the pinned arena of esmb200_layer_offload against the test's own packing at head widths 16, 24, 32, 64 and 128.
"""
import ctypes

import pytest
import torch

import kernel_refs as kr
import stack_replay as sr

pytestmark = pytest.mark.gpu


def report(name, **kv):
    print("PARITY", name, " ".join(f"{k}={v:.3e}" for k, v in kv.items()), flush=True)


def esm_layers(E, H, n_layers, n_distinct, rotary, seed):
    """n_layers TransformerLayer slots cycling through n_distinct modules with oracle.weights parameters"""
    from esm_b200.model import TransformerLayer
    from oracle.weights import make_state_dict
    sd = make_state_dict(n_distinct, E, H, seed=seed)
    mods = []
    for i in range(n_distinct):
        p = f"layers.{i}."
        d = {k[len(p):]: v for k, v in sd.items() if k.startswith(p) and (rotary or "rot_emb" not in k)}
        layer = TransformerLayer(E, 4 * E, H, use_rotary_embeddings=rotary)
        layer.load_state_dict(d, strict=True)
        mods.append(layer.cuda())
    return [mods[i % n_distinct] for i in range(n_layers)]


def padding(B, T, lengths):
    pad = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lengths):
        pad[b, n:] = True
    return pad


def offload(layers):
    """each distinct layer packed into its own pinned host buffer (cpu_offload()'s protocol, parameters left on the
    device)"""
    from esm_b200 import _lib
    lib = _lib.load()
    hosts = []
    for layer in {id(l): l for l in layers}.values():
        n = lib.esmb200_layer_packed_bytes(layer.embed_dim, layer.attention_heads, layer.ffn_embed_dim, layer.precision)
        host = torch.empty(n, dtype=torch.uint8, pin_memory=True)
        layer._binding.offload(torch.device("cuda", torch.cuda.current_device()), host)
        layer.handle()
        hosts.append(host)
    return hosts


def replay_stack(layers, x0, pad, T, cos, sin, precision, reprs, attn, stages, label, contacts=None,
                 zero_pad_rows=False):
    """Replays the stack layer by layer from x0 [B,T,E]; asserts each layer's output equals reprs[i] and the
    probabilities of the layers in attn equal the stack's, bit for bit (zero_pad_rows: the stack wrote the rows of padded
    query tokens as zeros); with stages (True: every layer, or a collection of layer indices), checks every stage of
    those layers against float64 and prints one PARITY line per stage with the worst ratio over the layers.  Returns the
    replayed final stream."""
    B, _, E = x0.shape
    H = layers[0].attention_heads
    M = B * T
    pad8 = pad.to(torch.uint8).contiguous()
    x = x0.clone().view(M, E)
    packs, worst = {}, {}
    for i, layer in enumerate(layers):
        pk = packs.get(id(layer))
        if pk is None:
            pk = packs[id(layer)] = sr.pack_esm(layer, precision)
        want_probs = i in attn or contacts is not None
        probs = torch.empty(B, H, T, T, device="cuda") if want_probs else None
        st = sr.replay_esm(layer, pk, x, pad8, B, T, cos, sin, precision, probs)
        if contacts is not None:
            contacts(i, probs)
        check_here = stages is True or (stages and i in stages)
        if check_here and precision == 2:
            sr.check_fp8_stages(layer, pk, st, pad, B, T, cos, sin, worst, probs if i in attn else None)
        elif check_here:
            sr.check_esm_stages(layer, pk, st, pad, B, T, cos, precision, worst, probs if i in attn else None, sin)
        assert torch.equal(x, reprs[i].view(M, E)), f"{label}: layer {i} output differs from the replay"
        if i in attn:
            if zero_pad_rows:
                probs.masked_fill_(pad[:, None, :, None], 0.0)
            assert torch.equal(probs, attn[i]), f"{label}: layer {i} probabilities differ from the replay"
        del st
    for name, r in worst.items():
        report(f"stack stage {label} {name}", worst_over_layers=r)
    for name, r in worst.items():
        assert r <= 1.0, (label, name, r)
    return x.view(B, T, E)


def run_esm(label, E, H, n_layers, n_distinct, T, lengths, precision, rotary, attn_at=(), stages=True,
            offloaded=False, pdl=False, contacts_only=False, seed=0):
    from esm_b200 import _lib
    from esm_b200.model import rope_tables, run_stack
    B = len(lengths)
    layers = esm_layers(E, H, n_layers, n_distinct, rotary, seed)
    for layer in layers:
        layer.precision = precision
    hosts = offload(layers) if offloaded else None
    pad = padding(B, T, lengths)
    x0 = torch.randn(B, T, E, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed + 1))
    inv = layers[0].self_attn.rot_emb.inv_freq if rotary else None
    cos, sin = rope_tables(inv, T) if rotary else (None, None)
    reprs = {i: torch.empty_like(x0) for i in range(n_layers)}
    x = x0.clone()
    lib = _lib.load()
    if pdl:
        _lib.check(lib.esmb200_set_option(b"pdl", 1))
    try:
        if contacts_only:
            # the store-free contact pass has no single-kernel entry point: its accumulators must equal those of the
            # storing pass (esmb200_stack_forward with every layer's maps and the same job), whose maps of the layers
            # in attn_at must equal the replay's
            job, bufs = contact_job(n_layers, H, B, T, precision)
            run_stack(layers, x, pad, cos, sin, reprs, [], zero_pad_rows=True, contact_job=job, contacts_only=True,
                      probs_scratch=bufs.get("scratch"))
            job2, bufs2 = contact_job(n_layers, H, B, T, precision)
            x2 = x0.clone()
            stored = run_stack(layers, x2, pad, cos, sin, None, list(range(n_layers)), zero_pad_rows=True,
                               contact_job=job2)
            torch.cuda.synchronize()
            assert torch.equal(x2, x)
            for k in ("acc", "row", "col"):
                assert torch.equal(bufs[k], bufs2[k]), f"{label}: contact {k} differs from the storing pass"
            attn = {i: stored[i] for i in attn_at}
            del stored
        else:
            attn = run_stack(layers, x, pad, cos, sin, reprs, list(attn_at))
        torch.cuda.synchronize()
    finally:
        if pdl:
            _lib.check(lib.esmb200_set_option(b"pdl", 0))
    # the replay's own rotary tables, built as rotary_embedding.py builds them
    rc, rs = sr.rope_ref(inv, T) if rotary else (None, None)
    xr = replay_stack(layers, x0, pad, T, rc, rs, precision, reprs, attn, stages, label, zero_pad_rows=contacts_only)
    assert torch.equal(x, xr), f"{label}: final stream differs from the replay"
    report(f"stack bit identity {label}", layers=n_layers, max_abs_diff=float((x - xr).abs().max()))
    for layer in {id(l): l for l in layers}.values():
        layer.release()
    del hosts


def contact_job(n_layers, H, B, T, precision, seed=3):
    """an esmb200_contact_job over positions [1, T-1) with random weights; its buffers by name"""
    from esm_b200 import _lib
    lo, hi = 1, T - 1
    S_ = hi - lo
    rb, cb, sb = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(_lib.load().esmb200_stack_contacts_bytes(n_layers, H, B, T, S_, precision, ctypes.byref(rb),
                                                        ctypes.byref(cb), ctypes.byref(sb)))
    g = torch.Generator(device="cuda").manual_seed(seed)
    bufs = dict(w=torch.randn(n_layers, H, device="cuda", generator=g), acc=torch.zeros(B, S_, S_, device="cuda"),
                row=torch.zeros(rb.value // 4, device="cuda"), col=torch.zeros(cb.value // 4, device="cuda"))
    if sb.value:
        bufs["scratch"] = torch.empty(sb.value // 4, device="cuda")
    job = _lib.ContactJob(bufs["w"].data_ptr(), None, bufs["acc"].data_ptr(), bufs["row"].data_ptr(),
                          bufs["col"].data_ptr(), lo, hi)
    return job, bufs


# ---- ESM-2 650M width ----------------------------------------------------------------------------------------------
LEN_1024 = [1024, 700, 333]


@pytest.mark.parametrize("precision", [0, 1, 2], ids=["fp16", "fp32x3", "fp8"])
def test_650m_stack_against_replay(precision):
    run_esm(f"650M p{precision} T=1024", 1280, 20, 33, 11, 1024, LEN_1024, precision, True, attn_at=(0, 16, 32))


@pytest.mark.parametrize("precision", [0, 1], ids=["fp16", "fp32x3"])
def test_650m_offloaded_stack_against_replay(precision):
    run_esm(f"650M offloaded p{precision} T=512", 1280, 20, 8, 3, 512, [512, 300], precision, True, attn_at=(1, 6),
            stages=False, offloaded=True, seed=5)


def test_650m_stack_with_pdl_against_replay():
    run_esm("650M pdl T=1024", 1280, 20, 8, 4, 1024, LEN_1024, 0, True, attn_at=(3,), stages=False, pdl=True, seed=7)


# ---- ESM-2 3B width ------------------------------------------------------------------------------------------------
def test_3b_contacts_stack_against_replay():
    run_esm("3B contacts p0 T=512", 2560, 40, 36, 4, 512, [512, 480, 129], 0, True, attn_at=(0, 35), contacts_only=True,
            seed=11)


def test_3b_fp8_stack_against_replay():
    run_esm("3B p2 T=512", 2560, 40, 36, 4, 512, [512, 200], 2, True, attn_at=(35,), seed=13)


# ---- ESM-1b --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("precision", [0, 1, 2], ids=["fp16", "fp32x3", "fp8"])
def test_esm1b_stack_against_replay(precision):
    run_esm(f"ESM-1b p{precision} T=1024", 1280, 20, 33, 11, 1024, [1024, 901, 17], precision, False, attn_at=(0, 32),
            seed=17)


# ---- esmb200_stack_contacts in fp32x3: the contact accumulators through esmb200_contact_accumulate -------------------
def test_split_stack_contacts_against_replay():
    from esm_b200 import _lib
    from esm_b200.model import rope_tables, run_stack
    E, H, n, T, lengths = 1280, 20, 6, 512, [512, 390]
    B = len(lengths)
    layers = esm_layers(E, H, n, 3, True, 19)
    for layer in layers:
        layer.precision = 1
    pad = padding(B, T, lengths)
    x0 = torch.randn(B, T, E, device="cuda", generator=torch.Generator(device="cuda").manual_seed(20))
    inv = layers[0].self_attn.rot_emb.inv_freq
    cos, sin = rope_tables(inv, T)
    reprs = {i: torch.empty_like(x0) for i in range(n)}
    job, bufs = contact_job(n, H, B, T, 1)
    x = x0.clone()
    run_stack(layers, x, pad, cos, sin, reprs, [], zero_pad_rows=True, contact_job=job, contacts_only=True,
              probs_scratch=bufs["scratch"])
    lo, hi = job.lo, job.hi
    S_ = hi - lo
    acc = torch.zeros_like(bufs["acc"])
    row = torch.zeros_like(bufs["row"])
    col = torch.zeros_like(bufs["col"])
    lib = _lib.load()
    nrow, ncol = B * H * S_, B * H * ((S_ + 15) // 16) * S_

    def fold(i, probs):
        probs.masked_fill_(pad[:, None, :, None], 0.0)  # padded query rows zero, as ESM2.forward asks
        sr.check(lib.esmb200_contact_accumulate(sr.P(probs), H * T * T, sr.P(bufs["w"][i]), None, sr.P(acc),
                                                sr.P(row[i * nrow:]), sr.P(col[i * ncol:]), B, H, T, lo, hi, sr.S()))

    rc, rs = sr.rope_ref(inv, T)
    xr = replay_stack(layers, x0, pad, T, rc, rs, 1, reprs, {}, False, "contacts p1", contacts=fold)
    torch.cuda.synchronize()
    assert torch.equal(x, xr)
    assert torch.equal(acc, bufs["acc"]) and torch.equal(row, bufs["row"]) and torch.equal(col, bufs["col"])
    report("stack bit identity contacts p1 T=512", layers=n, acc_max=float(acc.abs().max()))


# ---- ESM2.forward: the LM head and the final LayerNorm --------------------------------------------------------------
def test_forward_lm_head_against_replay():
    check_forward_lm_head("650M", 4, 1280, 20, seed=23)


def check_forward_lm_head(label, L_, E, H, seed):
    """ESM2.forward on three ragged sequences of up to 512 tokens against a replay of its layers and of the LM-head
    chain, bit for bit, and each stage of the chain against float64"""
    from esm_b200 import ESM2
    from oracle.weights import make_state_dict, make_tokens
    sd = make_state_dict(L_, E, H, seed=seed)
    model = ESM2(num_layers=L_, embed_dim=E, attention_heads=H)
    model.load_state_dict(sd, strict=True)
    model = model.eval().cuda()
    tokens = make_tokens([510, 301, 77], 512, seed=seed + 1, n_mask=3).cuda()
    out = model(tokens, repr_layers=[L_])
    B, T = tokens.shape
    M = B * T
    x = torch.empty(B, T, E, device="cuda")
    model._embed(tokens, x)
    pad = tokens.eq(model.padding_idx)
    pad8 = pad.to(torch.uint8)
    cos, sin = sr.rope_ref(model.layers[0].self_attn.rot_emb.inv_freq, T)
    xv = x.view(M, E)
    for layer in model.layers:
        sr.replay_esm(layer, sr.pack_esm(layer, 0), xv, pad8, B, T, cos, sin, 0)
    lib = sr.lib()
    ln, head = model.emb_layer_norm_after, model.lm_head
    a16 = torch.empty(M, E, dtype=torch.float16, device="cuda")
    sr.check(lib.esmb200_layernorm_f16(sr.P(xv), sr.P(ln.weight), sr.P(ln.bias), sr.P(a16), M, E, ln.eps, sr.S()))
    a16_pre = a16.clone()
    x_pre = xv.clone()
    h = torch.empty(M, E, device="cuda")
    w_dense = head.dense.weight.half()
    sr._gemm(kr.EPI_BIAS_GELU_F32, a16, w_dense, head.dense.bias, h, M, E, E, 0)
    hl = head.layer_norm
    sr.check(lib.esmb200_layernorm_f16(sr.P(h), sr.P(hl.weight), sr.P(hl.bias), sr.P(a16), M, E, hl.eps, sr.S()))
    V = head.weight.shape[0]
    w_out = torch.zeros(64, E, dtype=torch.float16, device="cuda")
    w_out[:V] = head.weight.half()
    b_out = torch.zeros(64, device="cuda")
    b_out[:V] = head.bias
    logits = torch.empty(M, 64, device="cuda")
    sr._gemm(kr.EPI_BIAS_F32, a16, w_out, b_out, logits, M, 64, E, 0)
    sr.check(lib.esmb200_layernorm(sr.P(xv), sr.P(ln.weight), sr.P(ln.bias), sr.P(xv), M, E, ln.eps, sr.S()))
    torch.cuda.synchronize()
    assert torch.equal(logits.view(B, T, 64)[:, :, :V], out["logits"])
    assert torch.equal(x, out["representations"][L_])
    # float64, each stage on the kernels' own operands: emb_layer_norm_after -> fp16, the dense layer's erf-GELU into
    # fp32, the head's LayerNorm -> fp16, the projection onto the vocabulary (the padded columns exact zeros) and the
    # in-place final LayerNorm (fp32)
    worst = {}
    sr.ln_stage(worst, "ln_after_f16", x_pre, ln, a16_pre, False)
    y, absdot = kr.gemm_exact(a16_pre, w_dense, head.dense.bias)
    b = 1.13 * kr.gemm_acc_bound(absdot, E, y) + kr.gelu_bound(y)
    worst["dense_gelu"] = sr._ratio((h.double() - kr.gelu64(y)).abs(), b)
    sr.ln_stage(worst, "head_ln_f16", h, hl, a16, False)
    y, absdot = kr.gemm_exact(a16, w_out[:V], b_out[:V])
    worst["logits"] = sr._ratio((logits[:, :V].double() - y).abs(), kr.gemm_acc_bound(absdot, E, y))
    assert bool((logits[:, V:] == 0).all())
    want, b = sr._ln_want(x_pre, ln)
    worst["final_ln"] = sr._ratio((xv.double() - want).abs(), b + kr.U32 * want.abs())
    for name, r in worst.items():
        report(f"stack stage lm_head {label} {name}", worst=r)
    for name, r in worst.items():
        assert r <= 1.0, (label, name, r)


# ---- MSA Transformer ------------------------------------------------------------------------------------------------
def axial_layers(n, seed):
    from esm_b200.msa import AxialTransformerLayer
    from oracle.msa_oracle import make_axial_state_dict
    sd = make_axial_state_dict(768, 3072, seed=seed, n_layers=n)
    out = []
    for i in range(n):
        p = f"layers.{i}."
        layer = AxialTransformerLayer(768, 3072, 12)
        layer.load_state_dict({k[len(p):]: v for k, v in sd.items() if k.startswith(p)}, strict=True)
        out.append(layer.cuda())
    return out


MSA_CASES = [(2, 32, 256, True, 0), (2, 32, 256, True, 1), (1, 6, 96, False, 0), (1, 6, 96, True, 1),
             (1, 17, 96, True, 0), (1, 17, 96, False, 1), (1, 128, 512, False, 0)]


@pytest.mark.parametrize("B,R,C,padded,precision", MSA_CASES,
                         ids=[f"{b}x{r}x{c}-{'pad' if p else 'nopad'}-p{q}" for b, r, c, p, q in MSA_CASES])
def test_axial_stack_against_maps_path_and_replay(B, R, C, padded, precision):
    from esm_b200.msa import run_axial_stack
    n = 12
    layers = axial_layers(n, seed=R + C)
    for layer in layers:
        layer.precision = precision
    E, H = 768, 12
    M = B * R * C
    pad = None
    if padded:
        pad = torch.zeros(B, R, C, dtype=torch.bool, device="cuda")
        pad[:, :, C - 19:] = True
        pad[B - 1, R - 2:] = True
    x0 = torch.randn(B, R, C, E, device="cuda", generator=torch.Generator(device="cuda").manual_seed(R))
    xa, xb, xr = x0.clone(), x0.clone(), x0.clone()
    stages = C <= 256  # the float64 stages at 2 x 32 x 256 and the R = 6 / 17 depths; 128 x 512 is bit identity only
    worst = {}
    for i, layer in enumerate(layers):
        ca = torch.full((B, C, H, R, R), float("nan"), device="cuda")
        ra = run_axial_stack([layer], xa, pad, row_attn_layers=[0], col_attn={0: ca})[0]
        rb, cb = layer.forward_batch_major(xb, pad, need_probs=True)
        rr = torch.empty(H, B, C, C, device="cuda")
        pk = sr.pack_axial(layer, precision)
        st = sr.replay_axial(layer, pk, xr.view(M, E), pad, B, R, C, precision, rr)
        torch.cuda.synchronize()
        assert torch.equal(xa, xb), f"layer {i}: run_axial_stack and forward_batch_major differ"
        assert torch.equal(xa, xr), f"layer {i}: run_axial_stack and the replay differ"
        assert torch.equal(ra, rb) and torch.equal(ra, rr), f"layer {i}: row attention maps differ"
        # forward_batch_major returns the reference's [H,C,B,R,R]; the stack's buffer is [B,C,H,R,R]
        assert torch.equal(cb, ca.permute(2, 1, 0, 3, 4)), f"layer {i}: column attention maps differ"
        del cb
        if stages:
            sr.check_axial_stages(layer, pk, st, pad, B, R, C, precision, worst, col_probs=ca)
        else:
            cpad = (pad.permute(0, 2, 1).reshape(B * C, R) if pad is not None else
                    torch.zeros(B * C, R, dtype=torch.bool, device="cuda"))
            assert not bool(ca.isnan().any()), f"layer {i}: a column map was not written"
            sr.column_zero_stage("col_probs", ca.view(B * C, H, R, R), cpad)
        del st, ca
    label = f"MSA {B}x{R}x{C} padded={padded} p{precision}"
    for name, r in worst.items():
        report(f"stack stage {label} {name}", worst_over_layers=r)
    for name, r in worst.items():
        assert r <= 1.0, (label, name, r)
    xs = x0.clone()
    run_axial_stack(layers, xs, pad)
    torch.cuda.synchronize()
    assert torch.equal(xs, xa), "the 12-layer call differs from the layer-by-layer calls"
    report(f"stack bit identity {label}", layers=n,
           row_scale=sr.q_scale(64, R))
    for layer in layers:
        layer.release()


# ---- the packed arena of an offloaded layer -------------------------------------------------------------------------
PACK_SHAPES = {16: (320, 20), 24: (480, 20), 32: (128, 4), 64: (256, 4), 128: (256, 2)}
PACK_CASES = [(d, p) for d, (E, H) in PACK_SHAPES.items() for p in (0, 1) if p == 0 or kr.fp32x3_accepts(E, H)]


@pytest.mark.parametrize("d,precision", PACK_CASES)
def test_offloaded_arena_equals_own_packing(d, precision):
    E, H = PACK_SHAPES[d]
    layer = esm_layers(E, H, 1, 1, True, seed=d)[0]
    layer.precision = precision
    hosts = offload([layer])
    torch.cuda.synchronize()
    want = sr.packed_arena(layer, precision == 1)
    assert hosts[0].numel() == want.numel()
    diff = int((hosts[0] != want).sum())
    report(f"packed arena d={d} E={E} H={H} p{precision}", bytes=float(want.numel()), differing=float(diff))
    assert diff == 0
    layer.release()
