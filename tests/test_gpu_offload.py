"""GPU: cpu_offload() streams the transformer layers' packed weights from pinned host memory through a two-slot device
ring (esmb200_stack_forward_streamed). The kernels and the packed bytes are those of the resident path, so every result
must be bit-identical (torch.equal) to the resident model on the same weights and tokens."""
import argparse
import ctypes
import gc

import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _sd(L, E, H, seed=0):
    from oracle.weights import make_state_dict
    return make_state_dict(L, E, H, seed=seed)


def _esm2(sd, L, E, H):
    from esm_b200 import ESM2
    m = ESM2(num_layers=L, embed_dim=E, attention_heads=H)
    m.load_state_dict(sd, strict=True)
    return m.eval()


def _pair(sd, L, E, H):
    """(resident, streamed) models with the same weights"""
    return _esm2(sd, L, E, H).to(DEV), _esm2(sd, L, E, H).cpu_offload(DEV)


def _repeated(n, E, H, seed=0):
    """ESM-2 whose ModuleList holds one seeded layer n times: the copy traffic of n layers, the memory of one"""
    m = _esm2(_sd(1, E, H, seed), 1, E, H)
    m.layers = nn.ModuleList([m.layers[0]] * n)
    m.num_layers = n
    return m


def _tokens(lengths, T, seed=3, n_mask=0):
    from oracle.weights import make_tokens
    return make_tokens(lengths, T, seed=seed, n_mask=n_mask).to(DEV)


def _assert_equal(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if k == "representations":
            assert a[k].keys() == b[k].keys()
            for i in a[k]:
                assert torch.equal(a[k][i], b[k][i]), f"representations[{i}]"
        else:
            assert torch.equal(a[k], b[k]), k


def test_650M_width_six_layers_every_output_and_masked_marginals():
    from esm_b200 import variants
    L, E, H = 6, 1280, 20
    res, st = _pair(_sd(L, E, H), L, E, H)
    assert all(layer.offloaded for layer in st.layers) and not any(layer.offloaded for layer in res.layers)
    tok = _tokens([300, 211, 97], 302, n_mask=4)
    kw = dict(repr_layers=list(range(L + 1)), return_contacts=True)
    _assert_equal(res(tok, **kw), st(tok, **kw))
    one = tok[2:3, :99]
    a = variants.masked_marginals(res, one, positions=list(range(1, 60)), max_tokens=2000)
    b = variants.masked_marginals(st, one, positions=list(range(1, 60)), max_tokens=2000)
    assert torch.equal(a, b)


def test_15B_width_three_distinct_layers_two_slot_heads():
    L, E, H = 3, 5120, 40
    res, st = _pair(_sd(L, E, H), L, E, H)
    tok = _tokens([298, 171], 300, n_mask=2)
    kw = dict(repr_layers=list(range(L + 1)), return_contacts=True)
    _assert_equal(res(tok, **kw), st(tok, **kw))


def test_esm1b_two_layers_learned_positions():
    from esm_b200 import ProteinBertModel
    from esm1b_weights import make_esm1b_state_dict
    L, E, H = 2, 256, 4
    args = argparse.Namespace(arch="roberta_large", layers=L, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                              max_positions=1024, emb_layer_norm_before=True, token_dropout=True)
    sd = make_esm1b_state_dict(L, E, H, seed=2)

    def build():
        m = ProteinBertModel(args, "roberta_large")
        m.load_state_dict(sd, strict=True)
        return m.eval()

    res, st = build().to(DEV), build().cpu_offload(DEV)
    tok = _tokens([400, 177], 402, n_mask=3)
    kw = dict(repr_layers=[0, 1, 2], return_contacts=True)
    _assert_equal(res(tok, **kw), st(tok, **kw))


def test_fp32x3_four_layers_650M_width_also_after_offload():
    L, E, H = 4, 1280, 20
    res, st = _pair(_sd(L, E, H), L, E, H)
    res.set_precision("fp32x3")
    st.set_precision("fp32x3")  # re-packs into a new arena of twice the size
    assert st._offload[1].numel() == L * 2 * 39_321_600
    tok = _tokens([255, 130], 257, n_mask=2)
    kw = dict(repr_layers=[2, 4], return_contacts=True)
    _assert_equal(res(tok, **kw), st(tok, **kw))


def test_half_model_with_host_parameters():
    L, E, H = 3, 640, 20
    sd = _sd(L, E, H, seed=4)
    res, st = _esm2(sd, L, E, H).half().cuda(), _esm2(sd, L, E, H).half().cpu_offload(DEV)
    assert st.layers[0].fc1.weight.dtype == torch.float16 and not st.layers[0].fc1.weight.is_cuda
    tok = _tokens([200, 90], 202)
    kw = dict(repr_layers=[1, 3], return_contacts=True)
    _assert_equal(res(tok, **kw), st(tok, **kw))


def _held_after_offload(build):
    """(torch tensors, the library's own allocations) on the device after cpu_offload(), in bytes.  torch's share is
    memory_allocated(): free memory (mem_get_info) alone also moves with the caching allocator's reuse of segments
    that earlier tests left partly in use.  The rest of the change in free memory is what the library allocated."""
    gc.collect()  # a layer and its binding reference each other
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    a0, r0, f0 = torch.cuda.memory_allocated(0), torch.cuda.memory_reserved(0), torch.cuda.mem_get_info(0)[0]
    m = build().cpu_offload(DEV)
    torch.cuda.synchronize()
    a1, r1, f1 = torch.cuda.memory_allocated(0), torch.cuda.memory_reserved(0), torch.cuda.mem_get_info(0)[0]
    del m
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return a1 - a0, (f0 - f1) - (r1 - r0)


def _assert_flat(name, few, many, extra_layers):
    mib = 1 << 20
    print(f"OFFLOAD {name}: torch {few[0] / mib:.2f} -> {many[0] / mib:.2f} MiB, "
          f"library {few[1] / mib:.2f} -> {many[1] / mib:.2f} MiB")
    assert many[0] - few[0] <= extra_layers * mib
    assert many[1] - few[1] <= extra_layers * mib + 2 * mib  # driver allocation granularity


def test_full_depth_15B_shape_48_layers_and_device_memory():
    E, H = 5120, 40
    _assert_flat("15B shape, 2 -> 48 repeats", _held_after_offload(lambda: _repeated(2, E, H)),
                 _held_after_offload(lambda: _repeated(48, E, H)), 46)
    _assert_flat("650M width, 2 -> 6 distinct layers", _held_after_offload(lambda: _esm2(_sd(2, 1280, 20), 2, 1280, 20)),
                 _held_after_offload(lambda: _esm2(_sd(6, 1280, 20), 6, 1280, 20)), 4)

    m = _repeated(48, E, H).cpu_offload(DEV)
    tok = _tokens([1022] * 4, 1024, n_mask=8)
    st = m(tok, repr_layers=[48])
    st = {"logits": st["logits"].clone(), "representations": {48: st["representations"][48].clone()}}
    m.cuda()  # ends the mode: the resident path again
    assert m._offload is None and not m.layers[0].offloaded and m.layers[0].fc1.weight.is_cuda
    res = m(tok, repr_layers=[48])
    assert torch.equal(res["representations"][48], st["representations"][48])
    assert torch.equal(res["logits"], st["logits"])


def test_ring_reuse_back_to_back_and_two_models_alternating():
    L, E, H = 4, 1280, 20
    sd1, sd2 = _sd(L, E, H, seed=5), _sd(L, E, H, seed=6)
    st1, st2 = _esm2(sd1, L, E, H).cpu_offload(DEV), _esm2(sd2, L, E, H).cpu_offload(DEV)
    ta, tb = _tokens([1000] * 16, 1002, seed=7), _tokens([700, 1000, 13] * 4, 1002, seed=8)
    alone = {}
    for name, m in (("1", st1), ("2", st2)):
        for tn, t in (("a", ta), ("b", tb)):
            alone[name + tn] = m(t, repr_layers=[L])["representations"][L].clone()
            torch.cuda.synchronize()
    ra = st1(ta, repr_layers=[L])["representations"][L]
    rb = st1(tb, repr_layers=[L])["representations"][L]  # no synchronisation in between
    torch.cuda.synchronize()
    assert torch.equal(ra, alone["1a"]) and torch.equal(rb, alone["1b"])
    outs = {name + tn: m(t, repr_layers=[L])["representations"][L]
            for tn, t in (("a", ta), ("b", tb)) for name, m in (("1", st1), ("2", st2))}
    torch.cuda.synchronize()
    for k, v in outs.items():
        assert torch.equal(v, alone[k]), k
    res1 = _esm2(sd1, L, E, H).to(DEV)
    assert torch.equal(res1(ta, repr_layers=[L])["representations"][L], alone["1a"])


def test_in_place_change_of_a_host_weight_is_picked_up():
    L, E, H = 3, 640, 20
    sd = _sd(L, E, H, seed=9)
    res, st = _pair(sd, L, E, H)
    tok = _tokens([250, 100], 252)
    before = st(tok)["logits"].clone()
    with torch.no_grad():
        for m in (res, st):
            m.layers[1].fc1.weight.mul_(1.25)
            m.layers[2].self_attn.q_proj.bias.add_(0.5)
    assert not st.layers[1].fc1.weight.is_cuda
    a, b = res(tok), st(tok)
    assert torch.equal(a["logits"], b["logits"])
    assert not torch.equal(b["logits"], before)


def test_resident_entry_points_refuse_an_offloaded_layer():
    from esm_b200 import _lib
    from esm_b200.model import _ptr, _stream
    L, E, H = 2, 256, 4
    st = _esm2(_sd(L, E, H), L, E, H).cpu_offload(DEV)
    lib = _lib.load()
    B, T = 2, 64
    x = torch.randn(B, T, E, device=DEV)
    x0 = x.clone()
    ws = torch.empty(lib.esmb200_workspace_bytes(E, H, 4 * E, B, T, 0), dtype=torch.uint8, device=DEV)
    handles = (ctypes.c_void_p * L)(*[layer.handle() for layer in st.layers])
    torch.cuda.synchronize()
    launches = lib.esmb200_launch_count()
    rc = lib.esmb200_stack_forward(handles, L, _ptr(x), None, B, T, None, None, None, None, 0, 0, None, _ptr(ws),
                                   ws.numel(), _stream())
    assert rc == -1 and b"layer 0 is offloaded" in lib.esmb200_last_error()
    rc = lib.esmb200_layer_forward(handles[1], _ptr(x), None, B, T, None, None, None, _ptr(ws), ws.numel(), _stream())
    assert rc == -1 and b"offloaded" in lib.esmb200_last_error()
    assert lib.esmb200_launch_count() == launches
    torch.cuda.synchronize()
    assert torch.equal(x, x0)
    # the streamed entry point refuses a resident layer and a ring smaller than two slots
    res = _esm2(_sd(L, E, H), L, E, H).to(DEV)
    ring = torch.empty(2 * lib.esmb200_layer_packed_bytes(E, H, 4 * E, 0), dtype=torch.uint8, device=DEV)
    copy = torch.cuda.Stream()
    args = (None, None, None, None, 0, 0, None, _ptr(ws), ws.numel())
    mixed = (ctypes.c_void_p * 2)(handles[0], res.layers[0].handle())  # packing the resident layer launches kernels
    torch.cuda.synchronize()
    launches = lib.esmb200_launch_count()
    rc = lib.esmb200_stack_forward_streamed(mixed, 2, _ptr(x), None, B, T, *args, _ptr(ring), ring.numel(),
                                            ctypes.c_void_p(copy.cuda_stream), _stream())
    assert rc == -1 and b"layer 1 is not offloaded" in lib.esmb200_last_error()
    rc = lib.esmb200_stack_forward_streamed(handles, L, _ptr(x), None, B, T, *args, _ptr(ring), ring.numel() - 1024,
                                            ctypes.c_void_p(copy.cuda_stream), _stream())
    assert rc == -1 and b"ring" in lib.esmb200_last_error()
    assert lib.esmb200_launch_count() == launches


def test_extract_cli_cpu_offload_writes_the_same_files(tmp_path):
    from esm_b200 import extract_cli
    L, E, H = 2, 128, 2
    sd = _sd(L, E, H)
    ckpt = tmp_path / "esm2_tiny.pt"
    torch.save({"cfg": {"model": {"encoder_layers": L, "encoder_embed_dim": E, "encoder_attention_heads": H,
                                  "token_dropout": True}},
                "model": {("encoder.sentence_encoder." + k): v for k, v in sd.items()}}, ckpt)
    g = torch.Generator().manual_seed(0)
    aas = "ACDEFGHIKLMNPQRSTVWY"
    fasta = tmp_path / "in.fasta"
    fasta.write_text("".join(f">p{i}\n" + "".join(aas[int(j)] for j in torch.randint(0, 20, (5 + 9 * i,), generator=g))
                             + "\n" for i in range(13)))
    tail = ["--toks_per_batch", "256", "--include", "mean", "per_tok", "bos", "contacts", "--repr_layers", "0", "1", "2"]
    p = extract_cli.create_parser()
    one, two = tmp_path / "resident", tmp_path / "offload"
    assert extract_cli.run(p.parse_args([str(ckpt), str(fasta), str(one)] + tail)) == 13
    assert extract_cli.run(p.parse_args([str(ckpt), str(fasta), str(two)] + tail + ["--cpu-offload"])) == 13
    files = sorted(f.name for f in one.glob("*.pt"))
    assert files == sorted(f.name for f in two.glob("*.pt")) and len(files) == 13
    for f in files:
        a, b = torch.load(one / f, weights_only=False), torch.load(two / f, weights_only=False)
        assert a["label"] == b["label"]
        for key in ("representations", "mean_representations", "bos_representations"):
            assert a[key].keys() == b[key].keys()
            for layer in a[key]:
                assert torch.equal(a[key][layer], b[key][layer]), (f, key)
        assert torch.equal(a["contacts"], b["contacts"]), f
