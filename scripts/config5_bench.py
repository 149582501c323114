"""BASELINE.json configs[4]: esm_msa1b_t12_100M axial (row + column) attention forward on a synthetic 128 x 512 MSA,
1xH100: 12 AxialTransformerLayers (E=768, H=12, F=3072), seeded random weights. Prints ms per MSA. Developer tool."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from esm_b200.msa import AxialTransformerLayer  # noqa: E402


def main():
    torch.manual_seed(0)
    layers = [AxialTransformerLayer(768, 3072, 12).eval().cuda() for _ in range(12)]
    R, C, B, E = 128, 512, 1, 768
    x = torch.randn(B, R, C, E, device="cuda")  # batch-major residual stream, as the model keeps it between layers

    def fwd():
        y = x.clone()
        for l in layers:
            l.forward_batch_major(y)  # in place
        return y
    for _ in range(2):
        y = fwd()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    n = 5
    for _ in range(n):
        y = fwd()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / n
    M = R * C
    flops = 12 * (8 * 2 * M * E * E + 2 * 2 * M * E * 3072 + 2 * 2 * 12 * C * C * R * 64 + 4 * C * 12 * R * R * 64)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    res = {"config": "12 x AxialTransformerLayer, MSA 128 x 512, E=768 H=12 (random init)", "ms_per_msa": round(ms, 3),
           "msa_per_s": round(1e3 / ms, 2), "TFLOP/s": round(flops / ms / 1e9, 1), "finite": bool(torch.isfinite(y).all())}
    # the whole model (embedding prologue, 12 layers, final LayerNorm, LM head) on tokens (1, 128, 512)
    from esm_b200 import pretrained
    model, _ = pretrained.esm_msa1b_t12_100M_UR50S(allow_random_init=True)
    model = model.cuda()
    gt = torch.Generator().manual_seed(1234)
    tokens = torch.randint(4, 24, (1, R, C), generator=gt)   # the 20 standard amino acids, <cls> in column 0, no padding
    tokens[:, :, 0] = 0
    tokens = tokens.cuda()
    for _ in range(2):
        out = model(tokens, repr_layers=[12])
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        out = model(tokens, repr_layers=[12])
    b.record()
    torch.cuda.synchronize()
    res["model_forward_ms_per_msa"] = round(a.elapsed_time(b) / n, 3)
    from esm_b200.msa import run_axial_stack
    xs = x.clone()
    run_axial_stack(layers, xs)
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        run_axial_stack(layers, xs)  # one esmb200_axial_stack_forward call for the 12 layers
    b.record()
    torch.cuda.synchronize()
    res["stack_single_call_ms_per_msa"] = round(a.elapsed_time(b) / n, 3)
    for _ in range(2):
        out = model(tokens, return_contacts=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        out = model(tokens, return_contacts=True)
    b.record()
    torch.cuda.synchronize()
    res["model_forward_with_contacts_ms_per_msa"] = round(a.elapsed_time(b) / n, 3)
    # where the time goes: torch profiler, top CUDA kernels of one forward
    try:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            fwd()
            torch.cuda.synchronize()
        tab = prof.key_averages().table(sort_by="cuda_time_total", row_limit=14, max_name_column_width=70)
        open(os.path.join(ROOT, "gpurun_out", "config5_profile.txt"), "w").write(tab)
        print(tab[-3500:])
    except Exception as e:  # profiler availability varies
        print("profiler unavailable:", e)
    print(json.dumps(res))
    json.dump(res, open(os.path.join(ROOT, "gpurun_out", "config5.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
