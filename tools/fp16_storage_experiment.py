"""CPU-only companion of tests/test_parity_experiment_gpu.py: how much of the tower's end-to-end deviation is inherent to
fp16 STORAGE of the two streams between stages, independent of any kernel?

The fp32 oracle tower (oracle/restate.py, same seed/weights as test_vldyhead_tower) is run a second time with the visual
stream rounded to fp16 after every stage (what any fp16 pipeline — including the reference under its own fp16 autocast,
engine/trainer.py:119-120 — stores), everything else in fp32.  Prints/records the deviation of the logits.

    python -m tools.fp16_storage_experiment > fp16_storage_amplification.json
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import restate  # noqa: E402  (test infrastructure; this tool is an experiment, not the product path)
from tools import synth  # noqa: E402

SIZES = [(20, 28), (10, 14), (5, 7), (3, 4), (2, 2)]


def rel(a, b):
    return (a - b).abs().max().item() / b.abs().max().item()


def tower(feats, hidden, masks, sd, nconv, round_v, round_ops):
    r16 = lambda t: t.half().float()  # noqa: E731
    v, h = restate.flatten_levels(feats), hidden
    if round_v:
        v = r16(v)
    for i in range(nconv):
        sdi = sd
        if round_ops:  # also round every weight matrix of the layer to fp16 (tensor-core operands)
            sdi = {k: (r16(t) if (k.startswith(f"dyhead_tower.{3 * i}") or k.startswith(f"dyhead_tower.{3 * i + 2}")) and t.dim() >= 2 else t)
                   for k, t in sd.items()}
        v, h = restate.bi_attention(v, h, masks, sdi, f"dyhead_tower.{3 * i}.b_attn.")
        if round_v:
            v = r16(v)
        h = restate.bert_layer(h, restate.extended_mask(masks), sdi, f"dyhead_tower.{3 * i + 1}.", clamp=50000.0)
        v = restate.flatten_levels(restate.dyconv(restate.split_levels(v, SIZES), sdi, f"dyhead_tower.{3 * i + 2}."))
        if round_v:
            v = r16(v)
    return restate.dot_product_head(v, h, sd), v, h


def main():
    torch.set_num_threads(8)
    gen = synth.Gen(78)
    nconv = 6
    sd = synth.vldyhead_sd(gen, nconv)
    B, T = 2, 256
    feats = [gen.randn(B, 256, h, w) for h, w in SIZES]
    hidden = gen.randn(B, T, 768)
    masks = torch.ones(B, T, dtype=torch.long)
    masks[0, 120:] = 0
    masks[1, 31:] = 0
    with torch.no_grad():
        lg0, v0, h0 = tower(feats, hidden, masks, sd, nconv, False, False)
        lg1, v1, h1 = tower(feats, hidden, masks, sd, nconv, True, False)
        lg2, v2, h2 = tower(feats, hidden, masks, sd, nconv, True, True)
    print(json.dumps({
        "what": "fp32 oracle tower vs the same oracle with fp16 storage of the visual stream between stages (CPU only)",
        "fp16_visual_storage": {"logits": rel(lg1, lg0), "visual": rel(v1, v0), "hidden": rel(h1, h0)},
        "fp16_visual_storage_and_fp16_weights": {"logits": rel(lg2, lg0), "visual": rel(v2, v0), "hidden": rel(h2, h0)},
    }, indent=1))


if __name__ == "__main__":
    main()
