"""GPU: vision-only evaluation of MQ-GLIP (VISION_QUERY.MASK_DURING_INFERENCE): the ``mask_prompt_tokens`` kernel against the
restatement (tests/vision_only_oracle.py, pinned to the reference by tests/test_vision_only_cpu.py), and every inference path with the
masking on against the same path with the masking off fed the restatement's masked ids."""
import random

import numpy as np
import pytest
import torch

import vision_only_oracle as vo
from util import assert_close

pytestmark = pytest.mark.gpu


def _set_bank(model, bank, no_rows=(), dev="cuda:0"):
    """A bank as torch.load returns it; the labels in ``no_rows`` get the reference's empty-list entry (no exemplar)."""
    sel = model.query_selector
    sel.query_bank = {k: ([] if k in no_rows else v.to(dev)) for k, v in bank.items()}
    sel.bank_version += 1


def _mode(model, on, rate=1.0):
    model.cfg.VISION_QUERY.MASK_DURING_INFERENCE = on
    model.cfg.VISION_QUERY.TEXT_DROPOUT = rate


@pytest.mark.parametrize("E,C", [(1, 7), (8, 80), (8 * 31, 40), (5, 0)])
def test_kernel_equals_restatement(dev, E, C):
    from mqdet_b200 import ops
    g = torch.Generator().manual_seed(E * 100 + C)
    T = 256
    ids = torch.randint(0, 30522, (E, T), generator=g)
    tok_cat = torch.randint(-1, C + 2, (E, T), generator=g).to(torch.int32)   # -1 and indices past C never mask
    flags = torch.randint(0, 2, (E, C), generator=g).to(torch.uint8)
    ids_d = ids.to(dev)
    out = ops.mask_prompt_tokens(ids_d, tok_cat.to(dev), flags.to(dev), 103)
    assert torch.equal(out.cpu(), vo.kernel(ids, tok_cat, flags, 103))
    assert torch.equal(ids_d.cpu(), ids)                  # out of place
    buf = torch.empty_like(ids_d)
    assert ops.mask_prompt_tokens(ids_d, tok_cat.to(dev), flags.to(dev), 7, out=buf) is buf
    assert torch.equal(buf.cpu(), vo.kernel(ids, tok_cat, flags, 7))


def _detector(dev, K=5):
    from oracle import synth
    from test_gcp_many_queries_gpu import _glip
    gen = synth.Gen(2024)
    sd = synth.detector_sd(gen, bias0=-1.5)
    ids, am, pmap = synth.prompt(10, 2, 256, gen)
    bank = synth.query_bank(pmap, K, gen)
    B, h, w = 2, 150, 203
    img = synth.images(gen, B, h, w)
    return _glip(sd, dev, K), sd, ids, am, pmap, bank, img, (h, w)


def _packed(model, il, caps, pmap):
    return model.forward_device(il, caps, pmap)["det_packed"].clone()


def test_forward_device_vision_only(dev):
    """TEXT_DROPOUT 1.0: packed rows bit-identical to the unmasked forward fed the restatement's ids; categories without
    queries keep their text; against the oracle; the flag off gives back the unmasked result; TEXT_DROPOUT 0.5 under a seed gives
    exactly the restatement's draws."""
    from mqdet_b200.structures.image_list import ImageList
    from oracle import restate
    model, sd, ids, am, pmap, bank, img, (h, w) = _detector(dev)
    B = img.shape[0]
    il = ImageList(img.to(dev), [(h, w)] * B)
    caps = {"input_ids": ids, "attention_mask": am}
    _set_bank(model, bank)
    plain = _packed(model, il, caps, pmap)
    no_rows = (3, 8)
    _set_bank(model, bank, no_rows)
    labels = list(pmap)
    has = vo.has_query(labels, model.query_selector.query_bank, 5)
    assert has.count(0) == 2
    _mode(model, True, 1.0)
    got = _packed(model, il, caps, pmap)
    masked = vo.forward_ids(ids[0], pmap, has, 1.0, B)
    for c in no_rows:
        assert torch.equal(masked[:, pmap[c]], ids[:, pmap[c]].expand(B, -1))
    assert (masked == vo.MASK_TOKEN_ID).sum().item() == B * sum(len(pmap[c]) for c in labels if c not in no_rows)
    _mode(model, False)
    want = _packed(model, il, {"input_ids": masked, "attention_mask": am.expand(B, -1).contiguous()}, pmap)
    assert torch.equal(got, want)
    # TEXT_DROPOUT 0.5: warm the state (the query selector's own draws), then the forward's draws equal the restatement's
    for seed in (1, 2):
        _mode(model, True, 0.5)
        model.forward_device(il, caps, pmap)    # the state cache holds one prompt state: toggling the flag rebuilds it
        random.seed(seed)
        got = _packed(model, il, caps, pmap)
        after = random.getstate()
        random.seed(seed)
        masked = vo.forward_ids(ids[0], pmap, has, 0.5, B)
        assert random.getstate() == after
        _mode(model, False)
        assert torch.equal(got, _packed(model, il, {"input_ids": masked, "attention_mask": am.expand(B, -1).contiguous()}, pmap))
    # the flag off: today's result
    _set_bank(model, bank)
    _mode(model, False, 1.0)
    assert torch.equal(_packed(model, il, caps, pmap), plain)
    # against the oracle's whole forward (every class has queries, so at 1.0 every class token is masked)
    _mode(model, True, 1.0)
    out = model.forward_device(il, caps, pmap)
    masked = vo.forward_ids(ids[0], pmap, [1] * len(labels), 1.0, B)
    ref = restate.detector(img, (h, w), masked, am, pmap, bank, sd)
    bad = []
    assert_close(out["head"]["hidden"], ref["fused_hidden"], 5e-3, "vision-only: fused language stream", defer=bad)
    assert_close(out["head"]["dot_product_logits"], ref["logits"], 1.5e-2, "vision-only: dot-product logits", defer=bad)
    assert not bad, bad


def test_forward_device_vision_only_no_host_sync(dev):
    from mqdet_b200.structures.image_list import ImageList
    model, sd, ids, am, pmap, bank, img, (h, w) = _detector(dev)
    model.query_selector.set_query_bank(bank)
    _mode(model, True, 1.0)
    il = ImageList(img.to(dev), [(h, w)] * img.shape[0])
    caps = {"input_ids": ids.to(dev), "attention_mask": am.to(dev)}
    model.forward_device(il, caps, pmap)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        model.forward_device(il, caps, pmap)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_inference_engine_replay_vision_only(dev):
    from mqdet_b200.engine.inference import InferenceEngine
    from mqdet_b200.structures.image_list import ImageList
    from oracle import synth
    model, sd, ids, am, pmap, bank, img, (h, w) = _detector(dev)
    _set_bank(model, bank, (2,))
    _mode(model, True, 1.0)
    gen = synth.Gen(99)
    B = 2
    caps = {"input_ids": ids, "attention_mask": am}
    batches = [synth.images(gen, B, h, w) for _ in range(3)]
    sizes = [(h, w)] * B
    want = [model(ImageList(b.to(dev), sizes), captions=caps, positive_map=pmap) for b in batches]
    eng = InferenceEngine(model, caps, pmap, tuple(batches[0].shape), sizes, use_graph=True, warmup=1)
    got = list(eng.run([b.pin_memory() for b in batches]))
    eng.close()
    for g_b, w_b in zip(got, want):
        for g, r in zip(g_b, w_b):
            assert len(g) == len(r) and len(r) > 0
            assert torch.equal(g.bbox.cpu(), r.bbox.cpu())
            assert torch.equal(g.get_field("scores").cpu(), r.get_field("scores").cpu())
            assert torch.equal(g.get_field("labels").cpu(), r.get_field("labels").cpu())
    _mode(model, True, 0.5)
    with pytest.raises(NotImplementedError, match="TEXT_DROPOUT"):
        InferenceEngine(model, caps, pmap, tuple(batches[0].shape), sizes)


def test_forward_chunked_vision_only(dev):
    """27 classes in chunks of 10, two images.  At 1.0: bit-identical to the unmasked chunked forward fed the masked chunk
    prompts.  At 0.5 under a seed: each (chunk, image) equals one forward of that chunk on that image fed the restatement's ids
    (drawn images outer, chunks inner), at the tolerance of the existing chunk-batching test.  Then LVIS fixed AP on the device."""
    from mqdet_b200.engine.lvis_eval import LvisEvaluatorFixedAP, LvisGroundTruth
    from mqdet_b200.structures.image_list import ImageList
    from test_lvis_eval_scale_gpu import _glip
    model, chunks, img, sizes = _glip(dev)
    sizes = [sizes[0]] * 2
    _set_bank(model, model.query_selector.query_bank, (4, 13, 21))
    il = ImageList(img.to(dev), sizes)
    caps = [{"input_ids": i, "attention_mask": a} for i, a, _ in chunks]
    pmaps = [pm for _, _, pm in chunks]
    bank = model.query_selector.query_bank
    has = [vo.has_query(list(pm), bank, 5) for pm in pmaps]
    _mode(model, True, 1.0)
    got = model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=2)["det_packed"].clone()
    m1 = vo.chunked_ids([(i[0], pm) for i, _, pm in chunks], has, 1.0, 1)
    _mode(model, False)
    mcaps = [{"input_ids": m1[c], "attention_mask": a} for c, (_, a, _) in enumerate(chunks)]
    assert torch.equal(got, model.forward_chunked_device(il, mcaps, pmaps, chunks_per_pass=2)["det_packed"])
    _mode(model, True, 0.5)
    model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=2)
    random.seed(4)
    got = model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=2)["det_packed"].cpu()
    random.seed(4)
    m5 = vo.chunked_ids([(i[0], pm) for i, _, pm in chunks], has, 0.5, 2)
    _mode(model, False)
    M = got.shape[2] - 1
    for c, (_, a, pm) in enumerate(chunks):
        for b in range(2):
            one = model.forward_chunked_device(ImageList(img[b:b + 1].to(dev), sizes[:1]), [{"input_ids": m5[c, b:b + 1], "attention_mask": a}],
                                               [pm], chunks_per_pass=1)["det_packed"][0, 0].cpu()
            n = int(one[M, 0])
            assert int(got[c, b, M, 0]) == n, (c, b)
            assert torch.equal(got[c, b, :n, 5], one[:n, 5])
            assert_close(got[c, b, :n, :5], one[:n, :5], 1e-4, f"chunk {c} image {b}")
    # LVIS fixed AP from the vision-only chunked output (README settings: MASK_DURING_INFERENCE True, TEXT_DROPOUT 1.0)
    _mode(model, True, 1.0)
    out = model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=2)
    pk = out["det_packed"].cpu()
    rng = np.random.default_rng(5)
    anns, images = [], []
    for b in range(2):
        for c in range(pk.shape[0]):
            for r in pk[c, b, :int(pk[c, b, M, 0]):3]:
                x1, y1, x2, y2 = (r[:4].numpy() + rng.normal(0, 2, 4)).tolist()
                bw, bh = max(x2 - x1, 1.0), max(y2 - y1, 1.0)
                anns.append({"id": len(anns) + 1, "image_id": b + 1, "category_id": int(r[5]), "bbox": [x1, y1, bw, bh],
                             "area": bw * bh, "iscrowd": 0})
        images.append({"id": b + 1, "width": sizes[b][1], "height": sizes[b][0], "neg_category_ids": [],
                       "not_exhaustive_category_ids": []})
    assert len(anns) > 3
    gt = {"images": images, "annotations": anns, "categories": [{"id": c, "frequency": "rcf"[c % 3]} for c in range(1, 28)]}
    ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, dev))
    ev.update_packed(out["det_packed"], [1, 2], out["image_sizes"], sizes)
    ev.accumulate()
    ev.summarize()
    assert 0.0 < ev.results["AP"] <= 1.0


def test_groundingdino_ignores_the_keys(dev):
    """MQ-GroundingDINO reads no masking key (the reference's groundingdino_new never does): outputs bit-identical with the flag."""
    from mqdet_b200.structures.image_list import ImageList
    from test_lvis_eval_scale_gpu import _gdino
    model, chunks, img, sizes = _gdino(dev)
    ids, am, pm = chunks[0]
    il = ImageList(img.to(dev), sizes)
    caps = {"input_ids": ids, "attention_mask": am}
    want = model.forward_device(il, caps, pm)["det_packed"].clone()
    wantc = model.forward_chunked_device(il, [caps], [pm])["det_packed"].clone()
    _mode(model, True, 1.0)
    assert torch.equal(model.forward_device(il, caps, pm)["det_packed"], want)
    assert torch.equal(model.forward_chunked_device(il, [caps], [pm])["det_packed"], wantc)
