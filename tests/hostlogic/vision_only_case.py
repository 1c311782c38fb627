"""Host-logic dry run of vision-only evaluation in ``GeneralizedVLRCNN_New`` (CPU, throw-away process): the prompt caches of
``forward_device`` / ``forward_chunked_device`` around a torch stand-in of ``ops.mask_prompt_tokens`` (the kernel's specification,
tests/vision_only_oracle.py).  It checks that the cache key follows MASK_DURING_INFERENCE / TEXT_DROPOUT, that at rate 1 the masked
ids are built once and reused, that below 1 every forward masks again from its own draws while the unmasked ids stay cached, that
Python's ``random`` advances by one draw per category per image per forward, and the configuration errors.

    python tests/hostlogic/vision_only_case.py
"""
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ops_double  # noqa: F401,E402  (patches mqdet_b200.ops; must come first)
import torch  # noqa: E402
from torch import nn  # noqa: E402

import vision_only_oracle as vo  # noqa: E402
from mqdet_b200 import ops  # noqa: E402
from mqdet_b200._lib import MqdetError  # noqa: E402
from mqdet_b200.config import mq_glip_t_cfg  # noqa: E402
from mqdet_b200.engine.inference import InferenceEngine  # noqa: E402
from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New  # noqa: E402
from mqdet_b200.modeling.query_selector.query_selector import QuerySelector  # noqa: E402

LAUNCHES = []


def mask_prompt_tokens(ids, tok_cat, flags, mask_id, out=None):
    LAUNCHES.append(tuple(ids.shape))
    assert ids.dtype == torch.int64 and tok_cat.dtype == torch.int32 and flags.dtype == torch.uint8
    assert tok_cat.shape == ids.shape and flags.shape[0] == ids.shape[0]
    return vo.kernel(ids, tok_cat, flags, mask_id)


ops.mask_prompt_tokens = mask_prompt_tokens


def model(rate, on=True):
    cfg = mq_glip_t_cfg(**{"MODEL.DEVICE": "cpu", "VISION_QUERY.MASK_DURING_INFERENCE": on, "VISION_QUERY.TEXT_DROPOUT": rate})
    m = GeneralizedVLRCNN_New.__new__(GeneralizedVLRCNN_New)   # only the prompt plumbing: no backbone, no head
    nn.Module.__init__(m)
    m.cfg, m.tokenizer, m._prompt = cfg, None, None
    m.rpn = nn.Module()
    m.rpn._tokmap = None
    m.query_selector = QuerySelector(cfg)
    return m


def set_bank(m, bank):
    """The bank as torch.load returns it: a class without exemplars holds an empty list (set_query_bank moves tensors only)."""
    m.query_selector.query_bank = dict(bank)
    m.query_selector.bank_version += 1


def prompt(n_cls, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(1, 256, dtype=torch.long)
    am = torch.zeros(1, 256, dtype=torch.long)
    pmap, pos = {}, 1
    for c in range(1, n_cls + 1):
        n = 1 + c % 3
        pmap[c] = list(range(pos, pos + n))
        ids[0, pos:pos + n] = torch.randint(1996, 29000, (n,), generator=g)
        pos += n + 1
    am[0, :pos] = 1
    bank = {c: ([] if c % 4 == 0 else torch.randn(3, 1, 8, generator=g)) for c in pmap}
    return {"input_ids": ids, "attention_mask": am}, pmap, bank


def draws_used(fn):
    """(result of fn, random.random() calls fn made) — by replaying the generator from a saved state."""
    st = random.getstate()
    out = fn()
    after = random.getstate()
    random.setstate(st)
    n = 0
    while random.getstate() != after:
        random.random()
        n += 1
        assert n < 100000
    return out, n


def main():
    B, C = 3, 9
    caps, pmap, bank = prompt(C, 0)
    labels = list(pmap)
    has = vo.has_query(labels, bank, 5)
    assert 0 < sum(has) < C
    ids0 = caps["input_ids"].clone()

    # rate 1: the masked ids are part of the cached state, built by one launch; each forward still draws B x C
    m = model(1.0)
    set_bank(m, bank)
    st = m._prompt_state(caps, pmap, B, torch.device("cpu"))
    assert LAUNCHES == [(B, 256)] and st["mask_rate"] == 1.0
    random.seed(3)
    want = vo.forward_ids(ids0[0], pmap, has, 1.0, B)
    for _ in range(3):
        got, n = draws_used(lambda: m._prompt_ids(m._prompt_state(caps, pmap, B, torch.device("cpu"))))
        assert n == B * C and torch.equal(got, want)
    assert len(LAUNCHES) == 1 and torch.equal(caps["input_ids"], ids0) and torch.equal(st["ids"], ids0.expand(B, -1))

    # the flag off: a new state (no stale masked ids), no draws, no launch; back on: masked again
    m.cfg.VISION_QUERY.MASK_DURING_INFERENCE = False
    st_off = m._prompt_state(caps, pmap, B, torch.device("cpu"))
    assert st_off is not st and st_off["mask_rate"] == 0.0
    got, n = draws_used(lambda: m._prompt_ids(st_off))
    assert n == 0 and torch.equal(got, ids0.expand(B, -1)) and len(LAUNCHES) == 1
    m.cfg.VISION_QUERY.MASK_DURING_INFERENCE = True
    got = m._prompt_ids(m._prompt_state(caps, pmap, B, torch.device("cpu")))
    assert torch.equal(got, want) and len(LAUNCHES) == 2

    # rate 0.5: a new state; every forward masks the cached unmasked ids with its own draws
    m.cfg.VISION_QUERY.TEXT_DROPOUT = 0.5
    st5 = m._prompt_state(caps, pmap, B, torch.device("cpu"))
    assert st5["mask_rate"] == 0.5 and "ids_masked" not in st5 and len(LAUNCHES) == 2
    random.seed(9)
    want = [vo.forward_ids(ids0[0], pmap, has, 0.5, B) for _ in range(4)]
    random.seed(9)
    for k in range(4):
        got, n = draws_used(lambda: m._prompt_ids(m._prompt_state(caps, pmap, B, torch.device("cpu"))))
        assert n == B * C and torch.equal(got, want[k]), k
    assert len(LAUNCHES) == 6 and torch.equal(st5["ids"], ids0.expand(B, -1))
    assert not all(torch.equal(want[0], w) for w in want[1:])

    # chunked: the key follows the rate too; at rate 1 the masked ids of each chunk are cached
    m.cfg.VISION_QUERY.TEXT_DROPOUT = 1.0
    c1 = m._chunk_state(caps, pmap, torch.device("cpu"))
    m.cfg.VISION_QUERY.MASK_DURING_INFERENCE = False
    c0 = m._chunk_state(caps, pmap, torch.device("cpu"))
    assert c1 is not c0 and c0["mask_rate"] == 0.0 and "ids_masked" not in c0
    assert torch.equal(c1["ids_masked"][0], vo.forward_ids(ids0[0], pmap, has, 1.0, 1)[0])
    m.cfg.VISION_QUERY.MASK_DURING_INFERENCE = True
    assert m._chunk_state(caps, pmap, torch.device("cpu")) is c1

    # configuration errors
    for key, val, exc in (("PURE_TEXT_RATE", 0.2, NotImplementedError), ("NEW_MASK_TOKEN", True, NotImplementedError)):
        bad = model(1.0)
        set_bank(bad, bank)
        setattr(bad.cfg.VISION_QUERY, key, val)
        try:
            bad._prompt_state(caps, pmap, B, torch.device("cpu"))
        except exc as e:
            assert key in str(e), e
        else:
            raise AssertionError(f"{key}={val} accepted")
    try:
        model(1.0)._prompt_state(caps, pmap, B, torch.device("cpu"))
    except MqdetError as e:
        assert "query bank" in str(e)
    else:
        raise AssertionError("vision-only evaluation without a bank accepted")
    half = model(0.5)
    set_bank(half, bank)
    try:
        InferenceEngine(half, caps, pmap, (B, 3, 64, 64), [(64, 64)] * B)
    except NotImplementedError as e:
        assert "TEXT_DROPOUT" in str(e)
    else:
        raise AssertionError("InferenceEngine accepted TEXT_DROPOUT 0.5")
    # nothing is masked with the flag off, whatever TEXT_DROPOUT says
    assert model(1.0, on=False).text_mask_rate() == 0.0
    print("PASS vision_only")


if __name__ == "__main__":
    main()
