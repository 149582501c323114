"""CPU study (no GPU): which fp16 roundings drive the error of the ESM-2 forward in the sharp-softmax regime.

Emulates the CUDA path's operand roundings inside the fp32 oracle (6 layers, 650M width, q/k weights x3) and switches
them off selectively: shows which roundings drive the error, and that full hi+lo operands ("fp32x3") restore
fp32-grade parity.   python scripts/precision_study.py [qk_gain]
"""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import esm2_oracle as O  # noqa: E402
from oracle.weights import make_state_dict, make_tokens  # noqa: E402

torch.set_num_threads(16)


def h(x):
    return x.half().float()


def hl(x):  # hi + lo split: 22 significand bits
    hi = x.half().float()
    return hi + (x - hi).half().float()


def ident(x):
    return x


def fwd(sd, L, H, tokens, cfg):
    pad = tokens.eq(1)
    x = O.embed(tokens, sd)
    mask = pad if pad.any() else None
    probs = []
    rest = cfg["rest"]
    for i in range(L):
        pre = f"layers.{i}."
        a = pre + "self_attn."
        xn = O.layer_norm(x, sd[pre + "self_attn_layer_norm.weight"], sd[pre + "self_attn_layer_norm.bias"])
        B, T, E = xn.shape
        d = E // H
        rq, rw, rqk = cfg["xn_qk"], cfg["w_qk"], cfg["qk"]
        q = (F.linear(rq(xn), rw(sd[a + "q_proj.weight"])) + sd[a + "q_proj.bias"]) * d ** -0.5
        k = F.linear(rq(xn), rw(sd[a + "k_proj.weight"])) + sd[a + "k_proj.bias"]
        v = F.linear(rest(xn), rest(sd[a + "v_proj.weight"])) + sd[a + "v_proj.bias"]
        q, k, v = (t.view(B, T, H, d).transpose(1, 2) for t in (q, k, v))
        cos, sin = O.rope_tables(sd[a + "rot_emb.inv_freq"], T)
        q, k = rqk(O.apply_rope(q, cos, sin)), rqk(O.apply_rope(k, cos, sin))
        v = rest(v)
        s = torch.matmul(q, k.transpose(-1, -2))
        if mask is not None:
            s = s.masked_fill(mask[:, None, None, :], float("-inf"))
        m = s.max(-1, keepdim=True).values
        e = torch.exp(s - m)
        o = (torch.matmul(cfg["p"](e), v) / e.sum(-1, keepdim=True)).transpose(1, 2).reshape(B, T, E)
        probs.append(torch.softmax(s, -1))
        x = x + F.linear(rest(o), rest(sd[a + "out_proj.weight"])) + sd[a + "out_proj.bias"]
        xn = O.layer_norm(x, sd[pre + "final_layer_norm.weight"], sd[pre + "final_layer_norm.bias"])
        hh = O.gelu(F.linear(rest(xn), rest(sd[pre + "fc1.weight"])) + sd[pre + "fc1.bias"])
        x = x + F.linear(rest(hh), rest(sd[pre + "fc2.weight"])) + sd[pre + "fc2.bias"]
    xf = O.layer_norm(x, sd["emb_layer_norm_after.weight"], sd["emb_layer_norm_after.bias"])
    return xf, torch.stack(probs, 1)


def main():
    L, E, H = 6, 1280, 20
    gain = float(sys.argv[1]) if len(sys.argv) > 1 else 3.0
    sd = make_state_dict(L, E, H, seed=0, qk_gain=gain)
    tokens = make_tokens([254, 180], 256, seed=5)
    print(f"6 layers, E=1280, H=20, qk_gain={gain}, tokens 2 x 256 (one padded to 180 residues); error vs the fp32 oracle")
    with torch.no_grad():
        ref = O.esm2_forward(sd, L, H, tokens, repr_layers=[L], need_head_weights=True)
        r, ra = ref["representations"][L], ref["attentions"]
        am = (~tokens.eq(1)).float()
        for name, cfg in [
            ("all MMA operands fp16 (the fp16 mode)", dict(xn_qk=h, w_qk=h, qk=h, p=h, rest=h)),
            ("q, k split hi+lo, everything else fp16 (r1 verdict's proposal)", dict(xn_qk=h, w_qk=h, qk=hl, p=h, rest=h)),
            ("q, k and Wq, Wk split", dict(xn_qk=h, w_qk=hl, qk=hl, p=h, rest=h)),
            ("q, k and LN output split", dict(xn_qk=hl, w_qk=h, qk=hl, p=h, rest=h)),
            ("whole logit path split (LN out, Wq, Wk, q, k)", dict(xn_qk=hl, w_qk=hl, qk=hl, p=h, rest=h)),
            ("logit path exact fp32, other operands fp16", dict(xn_qk=ident, w_qk=ident, qk=ident, p=h, rest=h)),
            ("every operand split hi+lo (the fp32x3 mode)", dict(xn_qk=hl, w_qk=hl, qk=hl, p=hl, rest=hl)),
        ]:
            x, a = fwd(sd, L, H, tokens, cfg)
            a = a * (am[:, None, None, :, None] * am[:, None, None, None, :])
            rel = float((x - r).norm() / r.norm())
            print(f"  {name:68s} repr rel_fro {rel:.2e}  max_abs {float((x - r).abs().max()):.2e}  "
                  f"attn max_abs {float((a - ra).abs().max()):.2e}")


if __name__ == "__main__":
    main()
