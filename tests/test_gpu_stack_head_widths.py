"""GPU (-m gpu): the layer stacks at the ESM-2 head widths other than 64 against the layer-by-layer replay of
tests/stack_replay.py, bit for bit, and every stage of the replay against float64 on its own inputs.

Heads of width d != 64 run in zero-padded 64-wide slots (one per head up to d = 64, two above): the QKV projection has
N = 3 Ea columns and out_proj K = Ea, Ea = 64 slots H, where E = d H.  At d = 16, 24 and 32 Ea is 1280 while E is 320,
480 and 640, so a stack that takes E for Ea (or the reverse) anywhere (GEMM shapes, workspace, ring slot maps, fp32x3
pitches, fp8 block scales over the padded rows) gives other bits than the replay, which packs the slots with its own map
(kernel_refs.slot_columns), scales q by fp32(d ** -0.5), pads its rotary tables past d/2 with other values than the
library's, and runs the QKV projection through esmb200_gemm_qkv_heads.  The float64 QKV stage runs in the reference's
layout (rotate-half over d/2 frequencies) and requires every padding column of q, k, v and ctx to be exactly 0.

Cases (random oracle.weights layers cycling through three distinct modules, an odd count so that the streamed ring's
slot parity does not follow layer identity; T = 1024, three ragged sequences, the models' depths and ffn_dim):
  * 8M width (E 320, H 20, d 16, 6 layers): fp16, fp32x3, fp8 (E = 320: a partial 128-wide K block) resident; fp16 and
    fp32x3 streamed; fp16 through esmb200_stack_contacts (120 channels);
  * 35M width (E 480, d 24, 12 layers): fp16, fp8 resident; fp16 streamed.  d = 24 is a width where fp32(1 / sqrt(d))
    is one ulp off the reference's q scale;
  * 150M width (E 640, d 32, 30 layers): fp16, fp32x3, fp8 resident; fp32x3 streamed;
  * 15B width (E 5120, H 40, d 128: two slots, two table halves, 48 layers): fp16, fp8 resident; fp16 streamed; fp16
    through esmb200_stack_contacts (1920 channels).  Stages at layers 0, 1, 2 and 47, bit identity at all 48;
  * ESM2.forward's LM head at the 35M and 8M widths, each stage against float64.
"""
import pytest

import test_gpu_stack_stages as ss

pytestmark = pytest.mark.gpu

LENGTHS = [1024, 700, 333]
T = 1024

# name: (E, H, layers)
WIDTHS = {"8M": (320, 20, 6), "35M": (480, 20, 12), "150M": (640, 20, 30), "15B": (5120, 40, 48)}
# (width, precision, streamed)
CASES = [("8M", 0, False), ("8M", 1, False), ("8M", 2, False), ("8M", 0, True), ("8M", 1, True),
         ("35M", 0, False), ("35M", 2, False), ("35M", 0, True),
         ("150M", 0, False), ("150M", 1, False), ("150M", 2, False), ("150M", 1, True),
         ("15B", 0, False), ("15B", 2, False), ("15B", 0, True)]
NAMES = ["fp16", "fp32x3", "fp8"]


def stages_of(width, n_layers):
    """the layers whose stages are checked: all, or at 15B width the first three and the last"""
    return (0, 1, 2, n_layers - 1) if width == "15B" else True


@pytest.mark.parametrize("width,precision,streamed", CASES,
                         ids=[f"{w}-{NAMES[p]}-{'streamed' if s else 'resident'}" for w, p, s in CASES])
def test_stack_at_head_width_against_replay(width, precision, streamed):
    E, H, n = WIDTHS[width]
    seed = 100 * (list(WIDTHS).index(width) + 1) + 10 * precision + streamed
    label = f"{width} d={E // H} p{precision}{' streamed' if streamed else ''} T={T}"
    ss.run_esm(label, E, H, n, 3, T, LENGTHS, precision, True, attn_at=(0, n - 1), stages=stages_of(width, n),
               offloaded=streamed, seed=seed)


@pytest.mark.parametrize("width", ["8M", "15B"])
def test_contacts_stack_at_head_width_against_replay(width):
    E, H, n = WIDTHS[width]
    ss.run_esm(f"{width} contacts d={E // H} p0 T={T}", E, H, n, 3, T, LENGTHS, 0, True, attn_at=(0, n - 1),
               stages=stages_of(width, n), contacts_only=True, seed=1000 + n)


@pytest.mark.parametrize("width", ["35M", "8M"])
def test_forward_lm_head_at_head_width_against_replay(width):
    E, H, _ = WIDTHS[width]
    ss.check_forward_lm_head(width, 4, E, H, seed=2000 + E)
