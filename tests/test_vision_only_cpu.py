"""CPU: vision-only evaluation (VISION_QUERY.MASK_DURING_INFERENCE).

tests/vision_only_oracle.py (the restatement the GPU tests compare against) is pinned to the reference's own code: the masking
block of maskrcnn_benchmark/modeling/detector/generalized_vl_rcnn_new.py (:397-407) compiled as it is, fed by the reference's own
``get_labels_and_maps_from_positive_map`` and ``QuerySelector``.  The masked ids and Python's ``random`` state after the draws
are recorded under tests/golden/vision_only_pins.pt, so that the comparison also runs where the reference is absent.  A host-logic
dry run (tests/hostlogic/vision_only_case.py) checks the detector's prompt caching around the masking."""
import ast
import os
import random
import subprocess
import sys
import textwrap
from types import SimpleNamespace as NS

import pytest
import torch

import refpin
import vision_only_oracle as vo
from oracle import ref_loader
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "vision_only_pins.pt")
REF_FILE = os.path.join("maskrcnn_benchmark", "modeling", "detector", "generalized_vl_rcnn_new.py")
T = 256
_store = None


def pinned(name, fn):
    """``refpin.pinned`` with the results in a file of their own (whole tensors)."""
    global _store
    if _store is None:
        _store = torch.load(PIN_FILE, weights_only=True) if os.path.exists(PIN_FILE) else {}
    if ref_loader.available():
        val = fn()
        if os.environ.get("MQDET_RECORD_PINS") == "1":
            _store[name] = refpin._shrink(val, True)
            torch.save(_store, PIN_FILE)
        return val
    assert name in _store, f"{name}: no recorded result in {PIN_FILE}"
    return refpin._expand(_store[name])


def _cfg(rate, k=3):
    return NS(MODEL=NS(DEVICE="cpu", LANGUAGE_BACKBONE=NS(MAX_QUERY_LEN=T)),
              VISION_QUERY=NS(ENABLED=True, TEXT_DROPOUT=rate, MASK_DURING_INFERENCE=True, PURE_TEXT_RATE=0.0, NEW_MASK_TOKEN=False,
                              QUERY_BANK_PATH="", LEARNABLE_BANK=False, ADD_VISION_LAYER=False, NUM_QUERY_PER_CLASS=k,
                              RANDOM_KSHOT=False))


def _prompt(seed, n_cls, empty=(), no_rows=()):
    """A caption of n_cls categories of 1-3 tokens each ('.' between them), a label with no token (skipped by the reference), and a
    bank where the labels in ``no_rows`` have no exemplar (the reference's empty-list entry)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(T, dtype=torch.long)
    ids[0] = 101
    pos, pmap, bank = 1, {}, {}
    for c in range(1, n_cls + 1):
        n = 1 + (c * 7 + seed) % 3
        pmap[c] = list(range(pos, pos + n))
        ids[pos:pos + n] = torch.randint(1996, 29000, (n,), generator=g)
        pos += n + 1
        ids[pos - 1] = 1012
        bank[c] = [] if c in no_rows else torch.randn(2 + c % 3, 1, 8, generator=g)
    ids[pos] = 102
    for c in empty:
        pmap[c] = []
        bank[c] = torch.randn(2, 1, 8, generator=g)
    return ids, pmap, bank


CASES = {   # name: (prompt seed, categories, empty labels, labels without rows, TEXT_DROPOUT, forwards, random seed)
    "p1_one": (0, 6, (), (2, 5), 1.0, 1, 10),
    "p1_three": (1, 9, (40,), (1, 4, 9), 1.0, 3, 11),
    "p05_one": (2, 7, (), (3,), 0.5, 1, 12),
    "p05_eight": (3, 12, (41,), (2, 7, 8, 11), 0.5, 8, 13),
    "p03_four": (4, 40, (), tuple(range(1, 41, 5)), 0.3, 4, 14),
}


def _state_tensor():
    version, words, gauss = random.getstate()
    assert version == 3 and gauss is None
    return torch.tensor(words, dtype=torch.int64)


def _reference(name):
    seed, n_cls, empty, no_rows, rate, n_img, rseed = CASES[name]
    ids, pmap, bank = _prompt(seed, n_cls, empty, no_rows)
    path = os.path.join(ref_loader.REF, REF_FILE)
    text = open(path).read()
    lines = text.splitlines()
    block = textwrap.dedent("\n".join(lines[396:407]))   # :397-407
    assert block.startswith("if (self.cfg.VISION_QUERY.ENABLED) and (self.cfg.VISION_QUERY.TEXT_DROPOUT > 0.)"), block[:80]
    assert block.rstrip().endswith("input_ids[i, position] = self.tokenizer.mask_token_id"), block[-80:]
    cls = next(n for n in ast.parse(text).body if isinstance(n, ast.ClassDef) and n.name == "GeneralizedVLRCNN_New")
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "get_labels_and_maps_from_positive_map")
    ns = {"torch": torch}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), ns)
    cfg = _cfg(rate)
    me = NS(cfg=cfg, training=False, tokenizer=NS(mask_token_id=vo.MASK_TOKEN_ID))
    labels, all_map = ns["get_labels_and_maps_from_positive_map"](me, pmap)
    sel = ref_loader.query_selector().QuerySelector(cfg)
    sel.query_bank = bank
    sel.eval()
    _, _, has = sel([labels], [all_map], None)
    code = compile(block, path, "exec")
    random.seed(rseed)
    out = []
    for _ in range(n_img):   # test-time forwards run one image each (:353)
        input_ids = ids[None].clone()
        exec(code, {"self": me, "input_ids": input_ids, "batched_all_map": [all_map], "batched_has_vision_query": has,
                    "batched_pos_category_map": None, "random": random, "torch": torch})
        out.append(input_ids[0])
    return {"ids": torch.stack(out), "state": _state_tensor(), "has": torch.tensor(has[0])}


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_reference(name):
    seed, n_cls, empty, no_rows, rate, n_img, rseed = CASES[name]
    ref = pinned(f"vision_only_{name}", lambda: _reference(name))
    ids, pmap, bank = _prompt(seed, n_cls, empty, no_rows)
    labels, _ = vo.token_rows(pmap, T)
    has = vo.has_query(labels, bank, 3)
    assert has == ref["has"].tolist()
    random.seed(rseed)
    got = vo.forward_ids(ids, pmap, has, rate, n_img)
    assert torch.equal(got, ref["ids"])
    assert torch.equal(_state_tensor(), ref["state"]), "Python random advanced differently"
    # every masked token belongs to a category with queries; at rate 1 each of them is masked, the rest keep their text
    _, rows = vo.token_rows(pmap, T)
    with_q = rows[torch.tensor(has, dtype=torch.bool)].any(0) if len(has) else torch.zeros(T, dtype=torch.bool)
    masked = got == vo.MASK_TOKEN_ID
    assert not (masked & ~with_q[None]).any()
    if rate >= 1:
        assert masked.eq(with_q[None]).all()
    else:
        assert 0 < int(masked.sum()) < int(with_q.sum()) * n_img


@pytest.mark.parametrize("name", sorted(CASES))
def test_detector_draws_and_tables_match_restatement(name):
    """The detector's host half (``draw_text_masks``, ``_mask_tables``' category table) against the restatement."""
    from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New as M
    seed, n_cls, empty, no_rows, rate, n_img, rseed = CASES[name]
    ids, pmap, bank = _prompt(seed, n_cls, empty, no_rows)
    labels, rows = vo.token_rows(pmap, T)
    has = vo.has_query(labels, bank, 3)
    random.seed(rseed)
    want = [vo.draw(has, rate) for _ in range(n_img)]
    random.seed(rseed)
    assert M.draw_text_masks([has] * n_img, rate) == want
    cat = torch.full((T,), -1, dtype=torch.int32)
    for j in range(rows.shape[0]):
        cat[rows[j]] = j
    flags = torch.tensor(want, dtype=torch.uint8)
    random.seed(rseed)
    assert torch.equal(vo.kernel(ids[None].expand(n_img, -1), cat[None].expand(n_img, -1), flags, vo.MASK_TOKEN_ID),
                       vo.forward_ids(ids, pmap, has, rate, n_img))


def test_chunked_draw_order():
    """Chunked prompts: image b of chunk c gets the draws of the reference's forward (image b, chunk c), images outer."""
    chunks, has = [], []
    for s in range(3):
        ids, pmap, bank = _prompt(20 + s, 5 + s, (), (1 + s,))
        chunks.append((ids, pmap))
        has.append(vo.has_query(vo.token_rows(pmap, T)[0], bank, 3))
    random.seed(5)
    got = vo.chunked_ids(chunks, has, 0.5, 2)
    random.seed(5)
    for b in range(2):
        for c, (ids, pmap) in enumerate(chunks):
            assert torch.equal(got[c, b], vo.forward_ids(ids, pmap, has[c], 0.5, 1)[0])


def test_config_defaults_and_rejections():
    from mqdet_b200.config import mq_glip_l_cfg, mq_glip_t_cfg, mq_groundingdino_t_cfg
    for f in (mq_glip_t_cfg, mq_glip_l_cfg, mq_groundingdino_t_cfg):
        vq = f().VISION_QUERY
        assert vq.MASK_DURING_INFERENCE is False and vq.NEW_MASK_TOKEN is False


def test_vision_only_host_logic():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostlogic", "vision_only_case.py")], capture_output=True,
                       text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "PASS vision_only" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])
