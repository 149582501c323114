"""BASELINE.json configs[3]: esm2_t36_3B_UR50D contact-prediction forward (need_head_weights=True), L=512, 1xH100.
Seeded random-init weights, B=16 (SURVEY §8d proposes 16; BASELINE.json leaves the batch open). Prints seq/s with and
without the attention/contact outputs. Developer/profile tool."""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from esm_b200 import pretrained  # noqa: E402


def main():
    B, T = int(os.environ.get("C4_B", 16)), 512
    model, alphabet = pretrained.load_model_and_alphabet("esm2_t36_3B_UR50D", allow_random_init=True)
    model = model.cuda()
    g = torch.Generator().manual_seed(1234)
    tok = torch.randint(4, 24, (B, T), generator=g)
    tok[:, 0] = 0
    tok[:, -1] = 2
    tok = tok.cuda()
    res = {}
    for name, kw in (("embed_only", dict(repr_layers=[36])), ("contacts", dict(repr_layers=[36], return_contacts=True))):
        for _ in range(2):
            out = model(tok, **kw)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        n = 3
        for _ in range(n):
            out = model(tok, **kw)
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / n
        res[name] = {"ms_per_batch": round(ms, 2), "seq_per_s": round(B / ms * 1e3, 2)}
        if "contacts" in out:
            res[name]["attentions_shape"] = list(out["attentions"].shape)
            res[name]["contacts_shape"] = list(out["contacts"].shape)
            res[name]["finite"] = bool(torch.isfinite(out["contacts"]).all())
        del out
        torch.cuda.empty_cache()
    if os.environ.get("C4_PROFILE"):
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = model(tok, repr_layers=[36], return_contacts=True)
            torch.cuda.synchronize()
        tab = prof.key_averages().table(sort_by="cuda_time_total", row_limit=14, max_name_column_width=60)
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        open(os.path.join(ROOT, "gpurun_out", "config4_profile.txt"), "w").write(tab)
        del out
    res["config"] = {"model": "esm2_t36_3B_UR50D (random init)", "B": B, "T": T}
    print(json.dumps(res))
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(res, open(os.path.join(ROOT, "gpurun_out", "config4.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
