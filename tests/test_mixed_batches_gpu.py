"""GPU: padded batches of differently sized images, as the reference's test loader forms them (TEST.IMS_PER_BATCH, BatchCollator ->
to_image_list).  The three kernels with per-image sizes (ATSS clip, query-update candidates, the test transform) bit for bit against
their one-size calls and restatements, the ATSS path also against the reference's own post-processor on a two-size batch; MQ-GLIP-T
on a four-size padded batch against one-image forwards at the same padded shape and against the oracle's detector;
``online_update`` over ``reference_test_batches`` against a host loop of padded forwards + extract_query; ``predict(mixed_sizes=True)``
into the COCO evaluator."""
import numpy as np
import pytest
import torch

import online_update_oracle as ou
import transform_oracle as to
from test_transform_gpu import GLIP, _cfg, _host_pipeline, _images
from util import assert_close

pytestmark = pytest.mark.gpu

LEVELS = [(20, 28), (10, 14), (5, 7), (3, 4), (2, 2)]
STRIDES = (8, 16, 32, 64, 128)
ASIZES = (64, 128, 256, 512, 1024)


def _atss_case(seed, E):
    from oracle import synth
    gen = synth.Gen(seed)
    _, _, pmap = synth.prompt(20, 2, 256, gen)
    N = sum(h * w for h, w in LEVELS)
    logits = gen.randn(E, N, 256, scale=1.5) - 2.0
    reg_ctr = torch.cat([gen.randn(E, N, 4, scale=1.5), gen.randn(E, N, 1, scale=2.0)], -1)
    return pmap, logits, reg_ctr


_ATSS_KEYS = ("det_packed", "num", "cand_totals", "level_counts")
_ATSS_CAND = ("cand_boxes", "cand_scores", "cand_labels")          # written up to cand_totals only


@pytest.mark.parametrize("chunks", [1, 3])
def test_atss_per_image_sizes_equal_one_image_calls(dev, chunks):
    """Element e = chunk * B + image clips to image (e % B)'s size; every output equals the one-element call with scalar sizes."""
    from mqdet_b200 import ops
    wh = [(221, 160), (160, 221), (97, 33), (224, 160)]
    B = len(wh)
    pmap, logits, reg_ctr = _atss_case(71 + chunks, B * chunks)
    lv = ops.Levels(LEVELS, dev)
    tm = ops.make_tokmap(pmap, 20, dev)
    scales = [1.0, 1.1, 1.2, 1.3, 1.4]
    lg, rc = logits.to(dev), reg_ctr.to(dev)
    r = ops.atss_postprocess(lg, rc, tm, lv, STRIDES, ASIZES, scales, [w for w, _ in wh], [h for _, h in wh], max_out=256)
    assert int(r["num"].min()) > 0
    clipped = 0
    for e in range(B * chunks):
        w, h = wh[e % B]
        one = ops.atss_postprocess(lg[e:e + 1].contiguous(), rc[e:e + 1].contiguous(), tm, lv, STRIDES, ASIZES, scales, float(w),
                                   float(h), max_out=256)
        for k in _ATSS_KEYS:
            assert torch.equal(r[k][e:e + 1], one[k]), (e, k)
        t = int(one["cand_totals"][0])
        for k in _ATSS_CAND:
            assert torch.equal(r[k][e, :t], one[k][0, :t]), (e, k)
        n = int(one["num"][0])
        boxes = one["det"][0, :n, :4].cpu()
        assert float(boxes[:, 0::2].max()) <= w - 1 and float(boxes[:, 1::2].max()) <= h - 1
        clipped += int((boxes[:, 2] == w - 1).sum() + (boxes[:, 3] == h - 1).sum())
    assert clipped > 0                                         # the per-image bound was reached, not only respected
    with pytest.raises(Exception, match="image sizes"):
        ops.atss_postprocess(lg[:3].contiguous(), rc[:3].contiguous(), tm, lv, STRIDES, ASIZES, scales, [1.0, 2.0], [1.0, 2.0])


def test_atss_two_size_batch_vs_reference_post_processor(dev):
    """ops.atss_postprocess with per-image sizes on the head outputs of a two-size padded batch against the reference's own
    ATSSPostProcessor on the same batch (recorded by tests/test_mixed_batches_cpu.py), image by image: the same detections, scores
    within the sigmoid's last bits and boxes within fp32 exp / decode rounding (the tolerances of tests/test_postprocess_gpu.py)."""
    import os
    import refpin
    from mqdet_b200 import ops
    from test_mixed_batches_cpu import ATSS_C, ATSS_IMAGE_HW, ATSS_LEVELS, ATSS_STRIDES, PIN_FILE, atss_two_size_inputs
    assert os.path.exists(PIN_FILE)
    ref = refpin._expand(torch.load(PIN_FILE, weights_only=True)["atss_two_sizes"])
    pmap, regs, ctrs, dots, _ = atss_two_size_inputs()
    B = len(ATSS_IMAGE_HW)
    logits = torch.cat(dots, 1)
    reg_ctr = torch.cat([torch.cat([r.permute(0, 2, 3, 1).reshape(B, -1, 4), c.reshape(B, -1, 1)], -1) for r, c in zip(regs, ctrs)], 1)
    lv = ops.Levels(ATSS_LEVELS, dev)
    r = ops.atss_postprocess(logits.to(dev), reg_ctr.contiguous().to(dev), ops.make_tokmap(pmap, ATSS_C, dev), lv, ATSS_STRIDES,
                             [8 * s for s in ATSS_STRIDES], [1.0] * len(ATSS_LEVELS), [w for _, w in ATSS_IMAGE_HW],
                             [h for h, _ in ATSS_IMAGE_HW])
    for b in range(B):
        want = ref[f"det{b}"]
        n = int(r["num"][b])
        assert n == want.shape[0], (b, n, want.shape[0])
        got = r["det"][b, :n].cpu()
        same = (want[:, None, 5] == got[None, :, 5]) & ((want[:, None, 4] - got[None, :, 4]).abs() <= 2e-6) & \
               ((want[:, None, :4] - got[None, :, :4]).abs().amax(-1) <= 2e-3)
        assert bool(same.any(1).all()) and bool(same.any(0).all()), f"image {b}: detections differ from the reference's"


def test_query_candidates_per_image_sizes_vs_restatement(dev):
    from mqdet_b200 import ops
    from test_online_update_gpu import _rows
    g = torch.Generator().manual_seed(5)
    wh = [(203, 150), (64, 48), (150, 203), (33, 97)]
    M = 60
    pk = torch.cat([_rows(g, 1, M, [M - 3 * b], s) for b, s in enumerate(wh)])
    bad = torch.zeros(1, dtype=torch.int32, device=dev)
    rois, labels, count = ops.query_candidates(pk.to(dev), wh, 0.6, 1.5, bad)
    n = int(count)
    want_b, want_l, want_i = [], [], []
    for b, s in enumerate(wh):
        boxes, lab = ou.candidates(pk[b], s, 0.6, 1.5)
        want_b.append(boxes), want_l.append(lab), want_i.append(torch.full((boxes.shape[0],), float(b)))
    assert n == sum(x.shape[0] for x in want_b) and int(bad) == 0
    assert torch.equal(rois[:n, 1:].cpu(), torch.cat(want_b)) and torch.equal(rois[:n, 0].cpu(), torch.cat(want_i))
    assert torch.equal(labels[:n].cpu().long(), torch.cat(want_l))
    one = ops.query_candidates(pk[:1].to(dev), [wh[0]], 0.6, 1.5, bad)   # a one-entry list is the one-size call
    ref = ops.query_candidates(pk[:1].to(dev), wh[0], 0.6, 1.5, bad)
    k = int(ref[2])
    assert int(one[2]) == k and torch.equal(one[0][:k], ref[0][:k]) and torch.equal(one[1][:k], ref[1][:k])


def test_mixed_transform_equals_host_pipeline(dev):
    """More than one launch of images (> 64), an image that keeps its size (shorter side = MIN_SIZE_TEST), extreme aspect ratios
    (MAX_SIZE_TEST binds), and small images whose tiles beyond their own size lie wholly in the padding."""
    from mqdet_b200.engine import transforms as tr
    size, max_size = 48, 120
    base = [(48, 64), (36, 52), (60, 45), (7, 300), (300, 7), (13, 17), (48, 48), (90, 31)]
    sizes = [base[i % len(base)] if i % 9 else (29 + i % 5, 41 + i % 7) for i in range(70)]
    images = _images(sizes, 31)
    targets = {to.get_size((w, h), size, max_size) for h, w in sizes}
    assert len(targets) > 5 and (48, 64) in targets                  # (48, 64) keeps its size
    want, resized = _host_pipeline(images, size, max_size, GLIP, 32)
    il, orig = tr.TestTransform(_cfg(GLIP, size, max_size))(images, dev, mixed_sizes=True)
    assert torch.equal(il.tensors.cpu(), want)
    assert il.image_sizes == [r.shape[:2] for r in resized] and orig == [(w, h) for h, w in sizes]
    assert any(h + 16 <= want.shape[-2] for h, _ in il.image_sizes)   # 16-row tiles wholly in an image's padding exist
    il2, _ = tr.TestTransform(_cfg(GLIP, size, max_size))(images[:2], dev, mixed_sizes=True, pad=False)
    assert tuple(il2.tensors.shape[-2:]) == (48, 69)
    with pytest.raises(Exception, match="want_resized"):
        tr.TestTransform(_cfg(GLIP, size, max_size))(images[:2], dev, mixed_sizes=True, want_resized=True)
    one = [images[0], images[0]]                                      # mixed_sizes on one target size: the one-size batch
    a, _ = tr.TestTransform(_cfg(GLIP, size, max_size))(one, dev)
    b, _ = tr.TestTransform(_cfg(GLIP, size, max_size))(one, dev, mixed_sizes=True)
    assert torch.equal(a.tensors, b.tensors) and a.image_sizes == b.image_sizes


# ---------------------------------------------------------------------------------------------------------------------
# MQ-GLIP-T on a padded batch of four sizes
# ---------------------------------------------------------------------------------------------------------------------
MIXED = [(128, 160), (96, 224), (160, 128), (150, 203)]


def _mixed_batch(dev):
    from mqdet_b200.structures.image_list import to_image_list
    from oracle import synth
    from test_online_update_gpu import _case
    model, caps, pmap, start, _, _ = _case("glip")
    model.set_query_bank({k: v.clone() for k, v in start.items()})
    gen = synth.Gen(404)
    imgs = [synth.images(gen, 1, h, w)[0][:, :h, :w].contiguous().to(dev) for h, w in MIXED]
    return model, caps, pmap, to_image_list(imgs, 32)


def test_glip_mixed_batch_equals_one_image_forwards(dev):
    """Image b of the padded batch equals the one-image forward of x[b:b+1] at the same padded shape with size (h_b, w_b)
    (tolerance of test_round2_gpu.py::test_batch8_equals_single_image_runs); likewise the chunked path, chunk by chunk."""
    from mqdet_b200.structures.image_list import ImageList
    model, caps, pmap, il = _mixed_batch(dev)
    assert tuple(il.tensors.shape[-2:]) == (160, 224) and il.image_sizes == MIXED
    out = model.forward_device(il, caps, pmap)
    lg, det, num = out["head"]["dot_product_logits"].clone(), out["det"].clone(), out["num"].clone()
    labels = sorted(pmap)
    chunks = [{k: pmap[k] for k in labels[:5]}, {k: pmap[k] for k in labels[5:]}]
    ck = model.forward_chunked_device(il, [caps, caps], chunks)["det_packed"].clone()
    lists = model(il, captions=caps, positive_map=pmap)
    assert int(num.min()) > 0
    for b, (h, w) in enumerate(MIXED):
        one = ImageList(il.tensors[b:b + 1], [(h, w)])
        o1 = model.forward_device(one, caps, pmap)
        assert_close(lg[b:b + 1], o1["head"]["dot_product_logits"], 1e-4, f"image {b}: mixed-batch logits vs single")
        k = int(num[b])
        assert k == int(o1["num"][0])
        assert_close(det[b, :k], o1["det"][0, :k], 1e-4, f"image {b}: detections")
        assert float(det[b, :k, 0:4:2].max()) <= w - 1 and float(det[b, :k, 1:4:2].max()) <= h - 1
        assert lists[b].size == (w, h) and len(lists[b]) == k
        c1 = model.forward_chunked_device(one, [caps, caps], chunks)["det_packed"]
        for g in range(2):
            n = int(ck[g, b, -1, 0])
            assert n == int(c1[g, 0, -1, 0]), (b, g)
            assert_close(ck[g, b, :n], c1[g, 0, :n], 1e-4, f"image {b} chunk {g}: detections")


def _oracle_detector(img, image_sizes, ids, am, pmap, bank, sd):
    """oracle/restate.detector over a padded batch of differently sized images: its batch elements are independent and an image's
    size enters only its clip, so image b is ``detector(img[b:b+1], image_sizes[b])`` at the batch's padded shape (for one size this
    is the one batched call)."""
    from oracle import restate
    runs = [restate.detector(img[b:b + 1], hw, ids, am, pmap, bank, sd) for b, hw in enumerate(image_sizes)]
    return {"logits": torch.cat([r["logits"] for r in runs]), "fused_hidden": torch.cat([r["fused_hidden"] for r in runs]),
            "detections": [r["detections"][0] for r in runs]}


def test_glip_mixed_batch_vs_oracle_detector(dev):
    """A four-size padded batch through MQ-GLIP-T (K = 5) against the oracle's detector with per-image sizes: the fused language
    stream and the detections with the tolerances of the existing detector checks (test_gcp_many_queries_gpu.py::
    test_detector_forward_100_queries).  The dot-product logits get 5e-2 of their largest magnitude instead of 1.5e-2: this synthetic
    model departs from the fp32 oracle by up to 0.085 on images with little or no padding (0.070 on an unpadded 160 x 224 image, above
    the 1.5e-2 bound of 0.051 for that image), and by 0.19 on the 2 x 2 level of the image padded from 96 to 160 rows (measured on an
    H100 80GB HBM3)."""
    from mqdet_b200.structures.image_list import ImageList, to_image_list
    from oracle import synth
    from test_detector_gpu import _iou
    from test_gcp_many_queries_gpu import _glip
    gen = synth.Gen(505)
    sd = synth.detector_sd(gen, bias0=-1.5)
    ids, am, pmap = synth.prompt(10, 2, 256, gen)
    bank = synth.query_bank(pmap, 5, gen)
    model = _glip(sd, dev, 5)
    model.query_selector.set_query_bank(bank)
    il = to_image_list([synth.images(gen, 1, h, w)[0][:, :h, :w].contiguous() for h, w in MIXED], 32)
    ref = _oracle_detector(il.tensors, il.image_sizes, ids, am, pmap, bank, sd)
    il = ImageList(il.tensors.to(dev), il.image_sizes)
    caps = {"input_ids": ids, "attention_mask": am}
    out = model.forward_device(il, caps, pmap)
    bad = []
    assert_close(out["head"]["hidden"], ref["fused_hidden"], 5e-3, "mixed batch: fused language stream", defer=bad)
    assert_close(out["head"]["dot_product_logits"], ref["logits"], 5e-2, "mixed batch: dot-product logits", defer=bad)
    assert not bad, bad
    res = model(il, captions=caps, positive_map=pmap)
    for b, (r, (h, w)) in enumerate(zip(res, MIXED)):
        rb, rs, rl = ref["detections"][b]
        assert r.size == (w, h) and len(r) >= min(100, rb.shape[0]) - 5 and rb.shape[0] > 0
        assert float(rb[:, 0::2].max()) <= w - 1 and float(rb[:, 1::2].max()) <= h - 1
        iou = _iou(rb, r.bbox)
        same = rl[:, None] == r.get_field("labels")[None]
        matched = ((iou > 0.9) & same & ((rs[:, None] - r.get_field("scores")[None]).abs() < 2e-2)).any(1)
        assert matched.float().mean().item() >= 0.85, f"image {b}: only {matched.float().mean().item():.2f} matched"


def test_glip_warm_mixed_forward_reads_nothing_on_the_host(dev):
    model, caps, pmap, il = _mixed_batch(dev)
    model.forward_device(il, caps, pmap)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = model.forward_device(il, caps, pmap)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert int(out["num"].min()) > 0


# ---------------------------------------------------------------------------------------------------------------------
# online_update over the reference's batches
# ---------------------------------------------------------------------------------------------------------------------
def _ref_images(kind, dev):
    """Landscape and portrait images of three sizes in dataset order, for reference_test_batches(..., 8, grouping on)."""
    from oracle import synth
    gen = synth.Gen(808)
    make = synth.images if kind == "glip" else synth.rgb_images
    sizes = [(150, 203), (203, 150), (128, 160), (150, 203), (160, 128), (128, 160), (150, 203), (203, 150), (128, 160), (150, 203),
             (150, 203), (128, 160)]
    return [make(gen, 1, h, w)[0][:, :h, :w].contiguous().to(dev) for h, w in sizes], sizes


def _host_loop_batches(kind, model, caps, pmap, start, batches):
    """Per batch: the padded forward, per-image BoxLists at each image's own size, scores > SCORE_THRESHOLD, extract_query
    (exclude_similar=True) with its expand_bbox; the bank installed at the start of every turn after the first."""
    from mqdet_b200.structures.bounding_box import BoxList
    vq = model.cfg.VISION_QUERY
    bank = ou.copy_bank(start)
    banks, kept_total = [], 0
    for turn in range(vq.NUM_TURNS):
        if turn > 0:
            model.set_query_bank({k: v.clone() for k, v in banks[-1].items()})
        for il in batches:
            if kind == "glip":
                out = model.forward_device(il, caps, pmap)
                pk = out["det_packed"].cpu()
            else:
                out = model.forward_chunked_device(il, [caps], [pmap])
                pk = out["det_packed"][0].cpu()
            pyr = out["pyramid16"]
            B = pk.shape[0]
            off, maps = 0, []
            for h, w in out["levels"].sizes:
                maps.append(pyr[:, off:off + h * w].float().transpose(1, 2).reshape(B, -1, h, w).contiguous())
                off += h * w
            kept = []
            for b, (h, w) in enumerate(il.image_sizes):
                n = int(pk[b, -1, 0])
                bl = BoxList(pk[b, :n, :4].clone(), (w, h), mode="xyxy")
                bl.add_field("scores", pk[b, :n, 4].clone())
                bl.add_field("labels", pk[b, :n, 5].long())
                kept.append(bl[bl.get_field("scores") > vq.SCORE_THRESHOLD])
            kept_total += sum(len(k) for k in kept)
            bank = model.extract_query(targets=kept, query_images=bank, visual_features=maps, exclude_similar=True,
                                       max_query_number=vq.MAX_TEST_QUERY_NUMBER)
        banks.append(ou.copy_bank(bank))
    return banks, kept_total


@pytest.mark.parametrize("kind", ["glip", "gdino"])
def test_online_update_over_reference_batches(dev, kind):
    from mqdet_b200.engine.batches import reference_test_batches
    from mqdet_b200.engine.online_update import make_batches, online_update
    from test_online_update_gpu import _assert_banks_equal, _prepare
    model, caps, pmap, start, _ = _prepare(kind)
    imgs, sizes = _ref_images(kind, dev)
    idx = reference_test_batches(sizes, 8, True)
    assert [len(b) for b in idx] == [8, 3, 1]
    batches = make_batches(imgs, 8, 32, orig_hw=sizes)
    assert [[tuple(imgs[i].shape[-2:]) for i in b] for b in idx] == [il.image_sizes for il in batches]
    assert len({tuple(s) for s in batches[0].image_sizes}) == 2
    want, kept = _host_loop_batches(kind, model, caps, pmap, start, batches)
    assert kept > 0
    model, caps, pmap, start, _ = _prepare(kind)
    res = online_update(model, batches, caps, pmap, model.cfg, bank=start)
    for t in range(3):
        _assert_banks_equal(res["banks"][t], want[t], f"{kind} turn {t}")
    _assert_banks_equal(res["eval_bank"], want[1], f"{kind} eval bank")
    rows = [sum(len(v) for v in b.values()) for b in [start] + want]
    assert rows[0] < rows[1], rows
    model, caps, pmap, start, _ = _prepare(kind)
    again = online_update(model, batches, caps, pmap, model.cfg, bank=start)
    for t in range(3):
        _assert_banks_equal(again["banks"][t], res["banks"][t], f"{kind} rerun turn {t}")


# ---------------------------------------------------------------------------------------------------------------------
# predict on a mixed-size set, scored by the COCO evaluator
# ---------------------------------------------------------------------------------------------------------------------
def test_predict_mixed_sizes_into_coco_eval(dev):
    from mqdet_b200.engine import transforms as tr
    from test_coco_eval_models_gpu import ORIG, _case, _check, _glip
    model, caps, pmap, _, _ = _glip(dev)
    model.cfg.INPUT.MIN_SIZE_TEST, model.cfg.INPUT.MAX_SIZE_TEST = 160, 224
    images = _images(ORIG, 23)                                   # (240, 336) -> (160, 224), (207, 285) -> (160, 220)
    il, orig = tr.TestTransform(model.cfg)(images, dev, mixed_sizes=True)
    assert il.image_sizes == [(160, 224), (160, 220)]
    host, _ = _host_pipeline(images, 160, 224, GLIP, 32)
    assert torch.equal(il.tensors.cpu(), host)
    out = model.forward_device(il, caps, pmap)
    boxlists = model(il, captions=caps, positive_map=pmap)
    res = tr.predict(model, images, caps, pmap, mixed_sizes=True)
    for r, q, (h, w) in zip(res, boxlists, ORIG):
        q = q.resize((w, h))
        assert r.size == (w, h) and torch.equal(r.bbox, q.bbox) and torch.equal(r.get_field("scores"), q.get_field("scores"))
    labels = sorted({int(v) for bl in boxlists for v in bl.get_field("labels").tolist()})
    assert len(labels) >= 3
    gt, l2c = _case(boxlists, labels)
    _check(gt, l2c, out["det_packed"], out["image_sizes"], boxlists, dev)
    assert np.isfinite(np.asarray(out["det_packed"].cpu())).all()
