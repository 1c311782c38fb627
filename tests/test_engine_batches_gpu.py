"""GPU: the reference's mixed-size test batches through the CUDA-graph engines (``run_batches`` / ``run_images``), one graph per
padded batch shape (B, Hp, Wp) with the image sizes read from a device table.  The ATSS clip with a device size table against the
by-value table (also under a captured graph whose table is rewritten), then MQ-GLIP-T and MQ-GroundingDINO-T engine results bit for
bit against the eager forward: over reference batches with a short tail, with sizes that differ at one padded shape, after another
batch size replaced the model's caches, under LRU eviction, from decoded uint8 images, and in vision-only evaluation."""
import random

import pytest
import torch

from test_mixed_batches_gpu import ASIZES, LEVELS, STRIDES, _atss_case, _ref_images

pytestmark = pytest.mark.gpu


def _same(got, want, what):
    assert len(got) == len(want), what
    for i, (g, r) in enumerate(zip(got, want)):
        assert g.size == r.size and len(g) == len(r), (what, i, g.size, r.size, len(g), len(r))
        assert torch.equal(g.bbox.cpu(), r.bbox.cpu()), (what, i)
        assert torch.equal(g.get_field("labels").cpu(), r.get_field("labels").cpu()), (what, i)
        assert torch.equal(g.get_field("scores").cpu(), r.get_field("scores").cpu()), (what, i)


def _glip():
    from test_online_update_gpu import _case
    model, caps, pmap, start, _, _ = _case("glip")
    model.set_query_bank({k: v.clone() for k, v in start.items()})
    return model, caps, pmap


def _il(imgs, dev):
    from mqdet_b200.structures.image_list import to_image_list
    return to_image_list([im.to(dev) for im in imgs], 32)


# ---------------------------------------------------------------------------------------------------------------------
# 1. the ATSS clip from a device size table
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_sizes,chunks", [(1, 1), (4, 1), (4, 3)])
def test_atss_device_sizes_equal_by_value_sizes(dev, n_sizes, chunks):
    from mqdet_b200 import ops
    wh = [(221, 160), (160, 221), (97, 33), (224, 160)][:n_sizes]
    E = 4 * chunks
    pmap, logits, reg_ctr = _atss_case(90 + n_sizes + chunks, E)
    lv = ops.Levels(LEVELS, dev)
    tm = ops.make_tokmap(pmap, 20, dev)
    scales = [1.0, 1.1, 1.2, 1.3, 1.4]
    lg, rc = logits.to(dev), reg_ctr.to(dev)
    table = torch.tensor([[float(w), float(h)] for w, h in wh], device=dev)
    by_value = ops.atss_postprocess(lg, rc, tm, lv, STRIDES, ASIZES, scales, [w for w, _ in wh], [h for _, h in wh], max_out=256)
    on_dev = ops.atss_postprocess(lg, rc, tm, lv, STRIDES, ASIZES, scales, table, None, max_out=256)
    assert int(by_value["num"].min()) > 0
    for k in ("det_packed", "num", "cand_totals", "level_counts"):
        assert torch.equal(on_dev[k], by_value[k]), k
    for e in range(E):
        t = int(by_value["cand_totals"][e])
        for k in ("cand_boxes", "cand_scores", "cand_labels"):
            assert torch.equal(on_dev[k][e, :t], by_value[k][e, :t]), (e, k)


def test_atss_graph_follows_rewritten_device_table(dev):
    """A graph captured with one table and replayed after the table is rewritten equals the eager call with the new sizes."""
    from mqdet_b200 import ops
    pmap, logits, reg_ctr = _atss_case(97, 4)
    lv = ops.Levels(LEVELS, dev)
    tm = ops.make_tokmap(pmap, 20, dev)
    scales = [1.0] * 5
    lg, rc = logits.to(dev), reg_ctr.to(dev)
    old = [(224.0, 160.0), (224.0, 160.0), (224.0, 160.0), (224.0, 160.0)]
    new = [(97.0, 33.0), (160.0, 221.0), (221.0, 160.0), (40.0, 90.0)]
    table = torch.tensor(old, device=dev)

    def call():
        return ops.atss_postprocess(lg, rc, tm, lv, STRIDES, ASIZES, scales, table, None, max_out=256)["det_packed"]

    call()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = call()
    table.copy_(torch.tensor(new))
    g.replay()
    want = ops.atss_postprocess(lg, rc, tm, lv, STRIDES, ASIZES, scales, [w for w, _ in new], [h for _, h in new], max_out=256)
    assert torch.equal(out, want["det_packed"])
    first = ops.atss_postprocess(lg, rc, tm, lv, STRIDES, ASIZES, scales, [w for w, _ in old], [h for _, h in old], max_out=256)
    assert not torch.equal(out, first["det_packed"])              # the new sizes did change the clip


# ---------------------------------------------------------------------------------------------------------------------
# 2-6, 8. MQ-GLIP-T through InferenceEngine.run_batches / run_images
# ---------------------------------------------------------------------------------------------------------------------
def test_glip_run_batches_over_reference_batches(dev):
    from mqdet_b200.engine.inference import InferenceEngine
    from mqdet_b200.engine.online_update import make_batches
    model, caps, pmap = _glip()
    imgs, sizes = _ref_images("glip", dev)
    batches = make_batches(imgs, 8, 32, orig_hw=sizes)
    assert [len(il.image_sizes) for il in batches] == [8, 3, 1]
    assert len(set(sizes)) >= 3 and any(h > w for h, w in sizes) and any(h < w for h, w in sizes)
    want = [model(il, captions=caps, positive_map=pmap) for il in batches]
    eng = InferenceEngine(model, caps, pmap)
    got = list(eng.run_batches(batches))
    for s, (g, w) in enumerate(zip(got, want)):
        _same(g, w, f"batch {s}")
    keys = {(len(il.image_sizes), *il.tensors.shape[-2:]) for il in batches}
    st = eng.batches.stats()
    assert st["captures"] == st["keys"] == len(keys) == 3
    pinned = [type(il)(il.tensors.cpu().pin_memory(), il.image_sizes) for il in batches]   # host batches, second pass
    again = list(eng.run_batches(pinned))
    assert eng.batches.stats()["captures"] == 3
    for s, (g, w) in enumerate(zip(again, want)):
        _same(g, w, f"second pass, batch {s}")
    eng.close()


def test_glip_sizes_are_not_baked_into_a_graph(dev):
    from mqdet_b200.engine.inference import InferenceEngine
    from mqdet_b200.structures.image_list import ImageList
    model, caps, pmap = _glip()
    imgs, sizes = _ref_images("glip", dev)
    a = _il([imgs[0], imgs[2]], dev)                              # (150, 203) + (128, 160) -> 160 x 224
    b = ImageList(a.tensors.flip(0).contiguous(), a.image_sizes[::-1])
    c = ImageList(a.tensors.clone(), [(120, 224), (160, 150)])    # the same pixels, other sizes
    assert tuple(a.tensors.shape) == tuple(b.tensors.shape) == (2, 3, 160, 224)
    want = [model(il, captions=caps, positive_map=pmap) for il in (a, b, c)]
    eng = InferenceEngine(model, caps, pmap)
    got = list(eng.run_batches([a, b, c]))
    assert eng.batches.stats()["captures"] == 1
    for s, (g, w) in enumerate(zip(got, want)):
        _same(g, w, f"batch {s}")
    assert [bl.size for bl in got[2]] == [(224, 120), (150, 160)]
    assert any(len(x) != len(y) or not torch.equal(x.bbox, y.bbox) for x, y in zip(got[0], got[2]))
    eng.close()


def test_glip_no_stale_caches_after_another_batch_size(dev):
    """Key A (B = 8), then key B (B = 3) replaces the model's single-entry caches; the freed blocks are handed out again and
    filled with NaN; a replay of A still equals eager."""
    from mqdet_b200.engine.inference import InferenceEngine
    from mqdet_b200.engine.online_update import make_batches
    model, caps, pmap = _glip()
    imgs, sizes = _ref_images("glip", dev)
    a, b, _ = make_batches(imgs, 8, 32, orig_hw=sizes)
    want_a = model(a, captions=caps, positive_map=pmap)
    eng = InferenceEngine(model, caps, pmap)
    list(eng.run_batches([a]))
    list(eng.run_batches([b]))
    junk = [torch.full((n,), float("nan"), device=dev) for n in (1 << 10, 1 << 14, 1 << 18, 1 << 20) for _ in range(32)]
    torch.cuda.synchronize()
    got = list(eng.run_batches([a]))[0]
    assert eng.batches.stats()["captures"] == 2
    _same(got, want_a, "replay of A after B")
    del junk
    eng.close()


def test_glip_eviction_at_one_graph(dev):
    from mqdet_b200.engine.inference import InferenceEngine
    from mqdet_b200.engine.online_update import make_batches
    model, caps, pmap = _glip()
    imgs, sizes = _ref_images("glip", dev)
    a, b, _ = make_batches(imgs, 8, 32, orig_hw=sizes)
    want = {id(a): model(a, captions=caps, positive_map=pmap), id(b): model(b, captions=caps, positive_map=pmap)}
    eng = InferenceEngine(model, caps, pmap, max_graphs=1)
    order = [a, b, a, a, b]
    got = list(eng.run_batches(order))
    for s, (il, g) in enumerate(zip(order, got)):
        _same(g, want[id(il)], f"batch {s}")
    st = eng.batches.stats()
    assert st["captures"] == 4 and st["evictions"] == 3 and st["live"] == 1 and st["keys"] == 2
    eng.close()


def test_glip_run_images_equals_predict(dev):
    from mqdet_b200.engine.batches import reference_test_batches
    from mqdet_b200.engine.inference import InferenceEngine
    from mqdet_b200.engine.transforms import predict
    from test_transform_gpu import _images
    model, caps, pmap = _glip()
    inp = model.cfg.INPUT
    saved = (inp.MIN_SIZE_TEST, inp.MAX_SIZE_TEST)
    inp.MIN_SIZE_TEST, inp.MAX_SIZE_TEST = 160, 224
    try:
        orig = [(240, 336), (207, 285), (336, 240), (240, 336), (300, 300), (207, 285), (285, 207), (240, 336), (207, 285),
                (240, 336), (336, 240)]
        images = _images(orig, 31)
        idx = reference_test_batches(orig, 8, True)
        assert len(idx) == 2 and min(len(i) for i in idx) < 8
        want = [predict(model, [images[i] for i in b], caps, pmap, mixed_sizes=True) for b in idx]
        eng = InferenceEngine(model, caps, pmap)
        got = list(eng.run_images(images, idx))
        for s, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f"batch {s}")
        assert got[0][0].size == (336, 240)
        eng.close()
    finally:
        inp.MIN_SIZE_TEST, inp.MAX_SIZE_TEST = saved


def test_glip_refuses_a_batch_larger_than_the_buffers(dev):
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.engine.inference import InferenceEngine
    from mqdet_b200.structures.image_list import ImageList
    model, caps, pmap = _glip()
    eng = InferenceEngine(model, caps, pmap)
    x = torch.zeros((9, 3, 32, 32), device=dev)
    with pytest.raises(MqdetError, match="exceeds the staging buffers"):
        list(eng.run_batches([ImageList(x, [(32, 32)] * 9)]))
    eng.close()


def test_glip_vision_only_run_batches_equals_eager(dev):
    from mqdet_b200.engine.inference import InferenceEngine
    from mqdet_b200.engine.online_update import make_batches
    model, caps, pmap = _glip()
    vq = model.cfg.VISION_QUERY
    saved = (vq.MASK_DURING_INFERENCE, vq.TEXT_DROPOUT)
    vq.MASK_DURING_INFERENCE, vq.TEXT_DROPOUT = True, 1.0
    try:
        imgs, sizes = _ref_images("glip", dev)
        batches = make_batches(imgs, 8, 32, orig_hw=sizes)
        random.seed(5)
        want = [model(il, captions=caps, positive_map=pmap) for il in batches]
        after_eager = random.getstate()
        vq.MASK_DURING_INFERENCE = False
        plain = model(batches[0], captions=caps, positive_map=pmap)
        vq.MASK_DURING_INFERENCE = True
        eng = InferenceEngine(model, caps, pmap)
        random.seed(5)
        got = list(eng.run_batches(batches))
        assert random.getstate() == after_eager                   # one draw per category and image, as the eager forwards
        for s, (g, w) in enumerate(zip(got, want)):
            _same(g, w, f"batch {s}")
        assert any(len(x) != len(y) or not torch.equal(x.bbox, y.bbox) for x, y in zip(got[0], plain))
        eng.close()
    finally:
        vq.MASK_DURING_INFERENCE, vq.TEXT_DROPOUT = saved
        model.invalidate_prompt_cache()


# ---------------------------------------------------------------------------------------------------------------------
# 7. MQ-GroundingDINO-T through GroundingDINOEngine.run_batches, one image per batch
# ---------------------------------------------------------------------------------------------------------------------
def test_gdino_run_batches_one_image_per_batch(dev):
    from mqdet_b200.engine.inference import GroundingDINOEngine
    from oracle import synth
    from test_online_update_gpu import _case
    model, caps, pmap, start, _, _ = _case("gdino")
    model.set_query_bank({k: v.clone() for k, v in start.items()})
    gen = synth.Gen(919)
    sizes = [(150, 203), (128, 160), (140, 210), (203, 150), (160, 224), (128, 160)]
    batches = [_il([synth.rgb_images(gen, 1, h, w)[0][:, :h, :w].contiguous()], dev) for h, w in sizes]
    shapes = {tuple(il.tensors.shape[-2:]) for il in batches}
    assert len(shapes) == 3 and len(set(sizes)) == 5
    want = [model(il, captions=caps, positive_map=pmap) for il in batches]
    eng = GroundingDINOEngine(model, caps, pmap)
    got = list(eng.run_batches(batches))
    for s, (g, w) in enumerate(zip(got, want)):
        _same(g, w, f"image {s}")
    assert sum(len(g[0]) for g in got) > 0
    st = eng.batches.stats()
    assert st["captures"] == st["keys"] == len(shapes)
    eng.close()
