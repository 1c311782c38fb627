"""GPU: chunked many-category (LVIS) evaluation through CUDA graphs.  ``forward_chunked_device(..., img_wh=...)`` of MQ-GLIP and
MQ-GroundingDINO against the host sizes (also under a captured graph whose size table is rewritten), the cached chunk-group state
and BERT prefix against a rebuild per pass, and ``ChunkedEngine`` bit for bit against eager ``forward_chunked``: one-image batches
of several sizes, after the chunk caches were cleared, under LRU eviction, from decoded uint8 images, in vision-only evaluation and
into the LVIS evaluator.  Five chunks at two chunks per pass, so the last pass is short."""
import random

import numpy as np
import pytest
import torch

from test_engine_batches_gpu import _same
from test_lvis_eval_scale_gpu import _gdino, _glip

pytestmark = pytest.mark.gpu

CPP = 2
SIZES = [(150, 203), (128, 160), (140, 210), (203, 150), (160, 224), (128, 160)]   # three padded shapes, two sizes at 160 x 224


def _chunk_prompts():
    from oracle import synth
    chunks = synth.chunked_prompts(27, 6, 256, synth.Gen(3303))     # 5 chunks (6, 6, 6, 6, 3 classes), labels 1..27
    return [{"input_ids": i, "attention_mask": a} for i, a, _ in chunks], [pm for _, _, pm in chunks]


@pytest.fixture(scope="module", params=["glip", "gdino"])
def case(request, dev):
    model = (_glip if request.param == "glip" else _gdino)(dev)[0]
    inp = model.cfg.INPUT
    saved = (inp.MIN_SIZE_TEST, inp.MAX_SIZE_TEST)
    inp.MIN_SIZE_TEST, inp.MAX_SIZE_TEST = 160, 224                 # staging buffers and run_images at this test's sizes
    caps, pmaps = _chunk_prompts()
    yield request.param, model, caps, pmaps
    inp.MIN_SIZE_TEST, inp.MAX_SIZE_TEST = saved


def _image(kind, gen, h, w, dev):
    from oracle import synth
    make = synth.images if kind == "glip" else synth.rgb_images
    return make(gen, 1, h, w)[0][:, :h, :w].contiguous().to(dev)


def _one_image_batches(kind, dev, sizes=SIZES, seed=919):
    from mqdet_b200.structures.image_list import to_image_list
    from oracle import synth
    gen = synth.Gen(seed)
    return [to_image_list([_image(kind, gen, h, w, dev)], 32) for h, w in sizes]


def _table(sizes, dev):
    return torch.tensor([[float(w), float(h)] for h, w in sizes], dtype=torch.float32, device=dev)


def _chunked(model, il, caps, pmaps, **kw):
    return model.forward_chunked_device(il, caps, pmaps, CPP, **kw)["det_packed"].clone()


# ---------------------------------------------------------------------------------------------------------------------
# 1-2. the model layer
# ---------------------------------------------------------------------------------------------------------------------
def test_img_wh_equals_host_sizes_and_follows_a_rewritten_table(case, dev):
    from mqdet_b200.structures.image_list import ImageList, to_image_list
    from oracle import synth
    kind, model, caps, pmaps = case
    gen = synth.Gen(77)
    il = to_image_list([_image(kind, gen, 160, 224, dev), _image(kind, gen, 138, 190, dev)], 32)
    want = _chunked(model, il, caps, pmaps)
    assert want.shape[:2] == (5, 2) and int(want[:, :, -1, 0].min()) > 0
    table = _table(il.image_sizes, dev)
    assert torch.equal(_chunked(model, il, caps, pmaps, img_wh=table), want)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = model.forward_chunked_device(il, caps, pmaps, CPP, img_wh=table)["det_packed"]
    keep = model.graph_state()
    new = [(120, 224), (160, 150)]
    table.copy_(_table(new, dev))
    g.replay()
    want_new = _chunked(model, ImageList(il.tensors, new), caps, pmaps)
    assert torch.equal(out, want_new)
    assert not torch.equal(want_new, want)                           # the new sizes did change the result
    g.reset()
    del keep


def test_cached_group_state_and_prefix_equal_a_rebuild_per_pass(case, dev):
    kind, model, caps, pmaps = case
    il = _one_image_batches(kind, dev, [(150, 203)])[0]
    model.cache_chunk_groups = False
    try:
        want = _chunked(model, il, caps, pmaps)
    finally:
        model.cache_chunk_groups = True
    first = _chunked(model, il, caps, pmaps)
    second = _chunked(model, il, caps, pmaps)                     # reads the cached prefix: an in-place write into it would show
    assert torch.equal(first, want) and torch.equal(second, want)
    assert int(want[:, :, -1, 0].min()) > 0


def test_an_empty_chunk_detects_nothing(case, dev):
    """A chunk with an empty positive map gets one score column without tokens, so it detects nothing, in a pass of its own or
    next to another chunk, and the other chunks' rows do not change; the engine replays such a pass as eager runs it.  Without a
    query bank, since the query selector has no class to pick queries for."""
    from mqdet_b200.engine.inference import ChunkedEngine
    kind, model, caps, pmaps = case
    il = _one_image_batches(kind, dev, [(150, 203)])[0]
    qs = model.query_selector
    bank = qs.query_bank
    qs.query_bank, qs.bank_version = None, qs.bank_version + 1
    try:
        want = model.forward_chunked_device(il, caps[:2], pmaps[:2], 1)["det_packed"].clone()
        assert int(want[:, :, -1, 0].sum()) > 0
        caps3, pmaps3 = [caps[0], caps[0], caps[1]], [pmaps[0], {}, pmaps[1]]
        for cpp in (1, 2):
            got = model.forward_chunked_device(il, caps3, pmaps3, cpp)["det_packed"]
            assert int(got[1, 0, -1, 0]) == 0, cpp
            if cpp == 1:
                assert torch.equal(got[[0, 2]], want)
        eng = ChunkedEngine(model, caps3, pmaps3, chunks_per_pass=1)
        _same(list(eng.run_batches([il]))[0], model.forward_chunked(il, caps3, pmaps3, 1), f"{kind} with an empty chunk")
        eng.close()
    finally:
        qs.set_query_bank(bank)


# ---------------------------------------------------------------------------------------------------------------------
# 3-7, 9. ChunkedEngine
# ---------------------------------------------------------------------------------------------------------------------
def test_run_batches_one_image_per_batch(case, dev):
    from mqdet_b200.engine.inference import ChunkedEngine
    kind, model, caps, pmaps = case
    batches = _one_image_batches(kind, dev)
    shapes = {tuple(il.tensors.shape) for il in batches}
    assert len(shapes) == 3 and len(set(SIZES)) == 5 and (1, 3, 224, 160) in shapes
    want = [model.forward_chunked(il, caps, pmaps, CPP) for il in batches]
    eng = ChunkedEngine(model, caps, pmaps, chunks_per_pass=CPP)
    got = list(eng.run_batches(batches))
    for s, (g, w) in enumerate(zip(got, want)):
        _same(g, w, f"{kind} image {s}")
    assert sum(len(g[0]) for g in got) > 0
    st = eng.stats()
    assert st["captures"] == st["keys"] == len(shapes)               # the sizes sharing 160 x 224 share one graph
    again = list(eng.run_batches([type(il)(il.tensors.cpu().pin_memory(), il.image_sizes) for il in batches]))
    assert eng.stats()["captures"] == len(shapes)
    for s, (g, w) in enumerate(zip(again, want)):
        _same(g, w, f"{kind} second pass, image {s}")
    eng.close()


def _tensors(obj, out):
    if torch.is_tensor(obj):
        out.append(obj)
    elif isinstance(obj, dict):
        for v in obj.values():
            _tensors(v, out)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            _tensors(v, out)
    return out


_GROUP_CACHES = ("_chunk_group_cache", "_chunk_text_cache")


def test_replay_after_the_chunk_caches_were_cleared(case, dev):
    """Capture at B = 1, then another batch size and chunk grouping clear the chunk and group caches, so only the graph holds
    the state it reads; the blocks freed by dropping the caches are handed out again and filled with NaN (checked: at least
    one is reused); a replay still equals eager."""
    from mqdet_b200.engine.inference import ChunkedEngine
    from mqdet_b200.structures.image_list import to_image_list
    from oracle import synth
    kind, model, caps, pmaps = case
    a = _one_image_batches(kind, dev, [(150, 203)])[0]
    want = model.forward_chunked(a, caps, pmaps, CPP)
    eng = ChunkedEngine(model, caps, pmaps, chunks_per_pass=CPP)
    list(eng.run_batches([a]))
    captured = {id(t) for e in eng.batches.graphs.values() for t in _tensors(e.state[-1], [])}
    gen = synth.Gen(5)
    two = to_image_list([_image(kind, gen, 128, 160, dev), _image(kind, gen, 96, 160, dev)], 32)
    model._chunk_cache.clear()
    model.CHUNK_GROUP_CAPACITY = 1                               # no room beside the new groups: the caches are cleared
    try:
        model.forward_chunked_device(two, caps, pmaps, 3)
    finally:
        del model.CHUNK_GROUP_CAPACITY
    cached = [model.__dict__.get(n) for n in _GROUP_CACHES]
    assert not captured & {id(t) for t in _tensors(cached, [])}     # the captured groups left the caches
    held = _tensors([cached, model._chunk_read, model.__dict__.get("_chunk_pass_cache"), model._chunk_cache], [])
    freed = {(t.untyped_storage().data_ptr(), t.untyped_storage().nbytes()) for t in held if not t.is_cpu and id(t) not in captured}
    del held, cached
    for n in _GROUP_CACHES + ("_chunk_pass_cache", "_chunk_cache"):
        model.__dict__.pop(n, None)
    model._chunk_read = None
    junk = [torch.full((max(n // 4, 1),), float("nan"), device=dev) for _, n in sorted(freed)]
    junk += [torch.full((n,), float("nan"), device=dev) for n in (1 << 10, 1 << 14, 1 << 18, 1 << 20) for _ in range(32)]
    spans = [(j.data_ptr(), j.data_ptr() + 4 * j.numel()) for j in junk]
    assert any(p < e and b < p + n for p, n in freed for b, e in spans), "no freed block was handed out again"
    torch.cuda.synchronize()
    got = list(eng.run_batches([a]))[0]
    assert eng.stats()["captures"] == 1
    _same(got, want, f"{kind} replay after the caches were cleared")
    del junk
    eng.close()


def test_more_chunk_groups_than_the_cache_capacity(case, dev):
    """One chunk per pass: 5 groups per forward against a capacity of 2.  The caches grow to one forward's groups instead of
    evicting inside it, so the capture finds them all cached and the replays equal eager."""
    from mqdet_b200.engine.inference import ChunkedEngine
    kind, model, caps, pmaps = case
    batches = _one_image_batches(kind, dev, [(150, 203), (203, 150)], seed=21)
    model.CHUNK_GROUP_CAPACITY = 2
    try:
        want = [model.forward_chunked(il, caps, pmaps, 1) for il in batches]
        eng = ChunkedEngine(model, caps, pmaps, chunks_per_pass=1)
        got = list(eng.run_batches(batches + batches))
        for s, (g, w) in enumerate(zip(got, want + want)):
            _same(g, w, f"{kind} one chunk per pass, batch {s}")
        assert eng.stats()["captures"] == 2
        cache = model.__dict__[_GROUP_CACHES[0] if kind == "glip" else _GROUP_CACHES[1]]
        assert len(cache) == 5
        eng.close()
    finally:
        del model.CHUNK_GROUP_CAPACITY


def test_reloaded_prefix_weights_rebuild_the_cached_prefix(case, dev):
    """The cached BERT prefix is keyed by its weights' (data_ptr, _version): after ``load_state_dict`` of changed embedding and
    layer-0 weights, a chunked forward equals one that rebuilds everything per pass."""
    kind, model, caps, pmaps = case
    il = _one_image_batches(kind, dev, [(150, 203)], seed=33)[0]
    before = _chunked(model, il, caps, pmaps)
    bert = model.language_backbone.body.model if kind == "glip" else model.bert
    prefix = {"embeddings.LayerNorm.bias": 0.2, "encoder.layer.0.output.dense.weight": 1.5}
    saved = {k: v.detach().clone() for k, v in bert.state_dict().items() if k in prefix}
    new = {k: (v + prefix[k] if k.endswith("bias") else v * prefix[k]) for k, v in saved.items()}
    try:
        bert.load_state_dict(new, strict=False)
        got = _chunked(model, il, caps, pmaps)
        model.cache_chunk_groups = False
        try:
            want = _chunked(model, il, caps, pmaps)
        finally:
            model.cache_chunk_groups = True
        assert torch.equal(got, want)
        assert not torch.equal(got, before)                          # the new weights did change the result
    finally:
        bert.load_state_dict(saved, strict=False)
    assert torch.equal(_chunked(model, il, caps, pmaps), before)


def test_lru_eviction_at_one_graph(case, dev):
    from mqdet_b200.engine.inference import ChunkedEngine
    kind, model, caps, pmaps = case
    a, b = _one_image_batches(kind, dev, [(150, 203), (203, 150)])
    want = {id(a): model.forward_chunked(a, caps, pmaps, CPP), id(b): model.forward_chunked(b, caps, pmaps, CPP)}
    eng = ChunkedEngine(model, caps, pmaps, chunks_per_pass=CPP, max_graphs=1)
    order = [a, b, a, a]
    for s, (il, g) in enumerate(zip(order, eng.run_batches(order))):
        _same(g, want[id(il)], f"{kind} batch {s}")
    st = eng.stats()
    assert st["captures"] == 3 and st["evictions"] == 2 and st["live"] == 1 and st["keys"] == 2
    eng.close()


def test_run_images_equals_transform_then_forward_chunked(case, dev):
    from mqdet_b200.engine.inference import ChunkedEngine
    from mqdet_b200.engine.transforms import TestTransform
    from test_transform_gpu import _images
    kind, model, caps, pmaps = case
    orig = [(240, 336), (207, 285), (336, 240), (300, 300)]
    images = _images(orig, 31)
    idx = [[i] for i in range(len(orig))]
    tf = TestTransform(model.cfg)
    want = []
    for i in range(len(orig)):
        il, o = tf([images[i]], dev, mixed_sizes=True)
        want.append([bl.resize(s) for bl, s in zip(model.forward_chunked(il, caps, pmaps, CPP), o)])
    eng = ChunkedEngine(model, caps, pmaps, chunks_per_pass=CPP)
    got = list(eng.run_images(images, idx))
    for s, (g, w) in enumerate(zip(got, want)):
        _same(g, w, f"{kind} image {s}")
    assert got[2][0].size == (240, 336)
    eng.close()


def test_engine_boxlists_into_the_lvis_evaluator(case, dev):
    from mqdet_b200.engine.inference import ChunkedEngine
    from mqdet_b200.engine.lvis_eval import LvisEvaluatorFixedAP, LvisGroundTruth
    kind, model, caps, pmaps = case
    batches = _one_image_batches(kind, dev, SIZES[:4], seed=12)
    eager = [model.forward_chunked(il, caps, pmaps, CPP)[0] for il in batches]
    eng = ChunkedEngine(model, caps, pmaps, chunks_per_pass=CPP)
    graphed = [r[0] for r in eng.run_batches(batches)]
    eng.close()
    rng = np.random.default_rng(3)
    anns, images = [], []
    for i, (bl, (h, w)) in enumerate(zip(eager, SIZES)):
        xyxy, labs = bl.bbox.numpy(), bl.get_field("labels").numpy()
        for k in range(0, len(labs), 3):
            x1, y1, x2, y2 = (xyxy[k] + rng.normal(0, 2, 4)).tolist()
            bw, bh = max(x2 - x1, 1.0), max(y2 - y1, 1.0)
            anns.append({"id": len(anns) + 1, "image_id": i + 1, "category_id": int(labs[k]), "bbox": [x1, y1, bw, bh],
                         "area": bw * bh, "iscrowd": 0})
        images.append({"id": i + 1, "width": w, "height": h, "neg_category_ids": [1, 2], "not_exhaustive_category_ids": []})
    assert len(anns) > 3
    gt = {"images": images, "annotations": anns, "categories": [{"id": c, "frequency": "rcf"[c % 3]} for c in range(1, 28)]}
    evs = []
    for lists in (eager, graphed):
        ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, dev))
        ev.update([(i + 1, {"boxes": bl.bbox.to(dev), "scores": bl.get_field("scores").to(dev), "labels": bl.get_field("labels").to(dev)})
                   for i, bl in enumerate(lists)])
        ev.accumulate()
        evs.append(ev)
    assert np.array_equal(evs[0].eval["precision"], evs[1].eval["precision"])
    assert np.array_equal(evs[0].eval["recall"], evs[1].eval["recall"])
    assert evs[0].summarize() == evs[1].summarize() and evs[0].results["AP"] > 0


# ---------------------------------------------------------------------------------------------------------------------
# 7-8. vision-only MQ-GLIP
# ---------------------------------------------------------------------------------------------------------------------
def _vision_only(model, rate):
    vq = model.cfg.VISION_QUERY
    saved = (vq.MASK_DURING_INFERENCE, vq.TEXT_DROPOUT)
    vq.MASK_DURING_INFERENCE, vq.TEXT_DROPOUT = True, rate
    return saved


def test_glip_vision_only_at_text_dropout_one(case, dev):
    from mqdet_b200.engine.inference import ChunkedEngine
    kind, model, caps, pmaps = case
    if kind != "glip":
        pytest.skip("vision-only evaluation (MASK_DURING_INFERENCE) is an MQ-GLIP path")
    batches = _one_image_batches(kind, dev, SIZES[:3])
    plain = model.forward_chunked(batches[0], caps, pmaps, CPP)
    saved = _vision_only(model, 1.0)
    try:
        model.forward_chunked(batches[0], caps, pmaps, CPP)      # the chunk states (and their query picks) of this rate, once
        random.seed(5)
        want = [model.forward_chunked(il, caps, pmaps, CPP) for il in batches]
        after_eager = random.getstate()
        eng = ChunkedEngine(model, caps, pmaps, chunks_per_pass=CPP)
        random.seed(5)
        got = list(eng.run_batches(batches))
        assert random.getstate() == after_eager                  # one draw per category, chunk and image, as the eager loop
        for s, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f"vision-only image {s}")
        assert len(got[0][0]) != len(plain[0]) or not torch.equal(got[0][0].bbox, plain[0].bbox)
        eng.close()
    finally:
        model.cfg.VISION_QUERY.MASK_DURING_INFERENCE, model.cfg.VISION_QUERY.TEXT_DROPOUT = saved


def test_glip_partial_text_dropout_is_refused(case, dev):
    from mqdet_b200.engine.inference import ChunkedEngine
    kind, model, caps, pmaps = case
    if kind != "glip":
        pytest.skip("vision-only evaluation (MASK_DURING_INFERENCE) is an MQ-GLIP path")
    saved = _vision_only(model, 0.5)
    try:
        with pytest.raises(NotImplementedError, match="TEXT_DROPOUT"):
            ChunkedEngine(model, caps, pmaps, chunks_per_pass=CPP)
    finally:
        model.cfg.VISION_QUERY.MASK_DURING_INFERENCE, model.cfg.VISION_QUERY.TEXT_DROPOUT = saved
