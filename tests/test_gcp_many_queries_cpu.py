"""CPU: the GCP restatement (oracle/restate.py) and QuerySelector with more than 16 vision queries per text token, pinned against the
reference's OWN MaskedCrossAttention (sparse), GatedCrossAttentionBlock, get_index_with_padding_batch and QuerySelector.  They run
live where the reference sources are present, else against the results recorded from them (tests/golden/gcp_many_queries_pins.pt;
float tensors above 1024 elements are kept as a seeded sample plus max |value|, see refpin.py)."""
import os
import random
import types

import numpy as np
import pytest
import torch

import refpin
from oracle import make_golden, ref_loader, restate, synth
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "gcp_many_queries_pins.pt")
_store = None


def pinned(name, fn):
    """``refpin.pinned`` with the results in a file of their own."""
    global _store
    if _store is None:
        _store = torch.load(PIN_FILE, weights_only=True) if os.path.exists(PIN_FILE) else {}
    if ref_loader.available():
        val = fn()
        if os.environ.get("MQDET_RECORD_PINS") == "1":
            _store[name] = refpin._shrink(val)
            torch.save(_store, PIN_FILE)
        return val
    assert name in _store, f"{name}: no recorded result in {PIN_FILE}"
    return refpin._expand(_store[name])


def many_query_case(S, T=32, ncls=4, D=768):
    """Three images, ``ncls`` classes with S queries each (so S = the most queries any token has): in image 0 class 0 keeps S // 3
    queries and class 1 keeps 3 (ragged banks); image 2 has no query at all; [CLS], separators and padding belong to no class."""
    gen = synth.Gen(4000 + S)
    sd = synth.gcp_block_sd(gen)
    _, _, pmap = synth.prompt(ncls, 2, T, gen)
    _, m = synth.vision_queries(pmap, S, T, D, gen)
    B = 3
    mask = m.expand(B, -1, -1).clone()
    mask[0, S // 3:S] = 0
    mask[0, S + 3:2 * S] = 0
    mask[2] = 0
    vision = gen.randn(B, mask.shape[1], D)
    x = gen.randn(B, T, D)
    return dict(sd=sd, x=x, vision=vision, mask=mask)


def _close(a, b, tol=2e-5):
    err, bmax = refpin.max_err(a, b)
    assert err <= tol * bmax + 1e-6, f"{err:.3e} (max|ref| {bmax:.3e})"


@pytest.mark.parametrize("S", [17, 32, 100])
def test_gcp_restatement_vs_reference_many_queries(S):
    c = many_query_case(S)
    assert int((c["mask"] != 0).sum(1).max()) == S

    def reference():
        m = ref_loader.modeling_bert_new()
        blk = m.GatedCrossAttentionBlock(dim=768, cfg=make_golden.ref_cfg()).eval()
        blk.load_state_dict(c["sd"], strict=True)
        with torch.no_grad():
            y = blk(c["x"], c["vision"], c["mask"])
            s = blk.attn(c["x"], c["vision"], c["mask"])
        idx = m.get_index_with_padding_batch(c["mask"].transpose(2, 1))
        return {"y": y, "s": s, "idx": idx}
    ref = pinned(f"gcp_many_queries_S{S}", reference)
    idx = restate.gcp_index(c["mask"])
    assert idx.shape[2] == S and refpin.equal(idx, ref["idx"])
    s = restate.gcp_sparse_attention(c["x"], c["vision"], c["mask"], c["sd"], "attn.")
    _close(s, ref["s"])
    _close(restate.gcp_block(c["x"], c["vision"], c["mask"], c["sd"]), ref["y"])
    # tokens of no class, and every token of the image without queries, get exactly zero attention output
    no_cls = c["mask"].sum(1) == 0
    assert no_cls[2].all() and s[no_cls].abs().max().item() == 0.0


def _vq_cfg(**over):
    vq = dict(QUERY_BANK_PATH="", LEARNABLE_BANK=False, ADD_VISION_LAYER=False, PURE_TEXT_RATE=0.0, NUM_QUERY_PER_CLASS=100,
              RANDOM_KSHOT=False)
    vq.update(over)
    return types.SimpleNamespace(MODEL=types.SimpleNamespace(DEVICE="cpu"), VISION_QUERY=types.SimpleNamespace(**vq))


@pytest.mark.parametrize("training,kshot,text_rate", [(False, False, 0.0), (True, True, 0.3)])
def test_query_selector_100_per_class_vs_reference(training, kshot, text_rate):
    """NUM_QUERY_PER_CLASS = 100 from banks of 150 rows per class (one class with 40): same tensors as the reference class."""
    from mqdet_b200.modeling.query_selector.query_selector import QuerySelector
    gen = synth.Gen(71)
    _, _, pmap = synth.prompt(12, 2, 256, gen)
    bank = synth.query_bank(pmap, 150, gen)
    bank[3] = bank[3][:40]
    labels = [sorted(bank.keys()), sorted(bank.keys())[::2]]
    T = 256
    loc = []
    for ls in labels:
        m = torch.zeros(len(ls), T)
        for i, c in enumerate(ls):
            m[i, torch.as_tensor(pmap[c])] = 1.0 / len(pmap[c])
        loc.append(m)
    cfg = _vq_cfg(RANDOM_KSHOT=kshot, PURE_TEXT_RATE=text_rate)

    def run(cls):
        sel = cls(cfg)
        sel.query_bank = {k: v.clone() for k, v in bank.items()}
        sel.train(training)
        np.random.seed(11)
        random.seed(12)
        return sel(labels, loc, [[1, 2, 3], [2]])
    ref = pinned(f"query_selector_k100_{int(training)}{int(kshot)}{int(text_rate > 0)}",
                 lambda: dict(zip(("q", "m", "h"), run(ref_loader.query_selector().QuerySelector))))
    q1, m1, h1 = run(QuerySelector)
    assert refpin.equal(q1, ref["q"]) and refpin.equal(m1, ref["m"]) and h1 == ref["h"]
    if not training:
        assert int((m1 != 0).sum(1).max()) == 100     # a class token attends to its 100 queries
