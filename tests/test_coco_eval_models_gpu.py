"""GPU: the COCO evaluator on real detector output.  ``update_packed`` on ``forward_device`` of a synthetic MQ-GLIP-T and
MQ-GroundingDINO-T (13-class prompt), and on ``forward_chunked_device`` of a chunked MQ-GLIP (G > 1 chunks), equals ``update``
on the BoxLists the models return and the restatement (tests/coco_eval_oracle.py) run on those BoxLists.  Labels go through a
``contiguous_category_id_to_json_id``-style table with gaps in the json ids and one label left out (its detections dropped);
the GT holds jittered copies of some detections, one of them crowd, at the GT image's size."""
import numpy as np
import pytest
import torch

import coco_eval_oracle as co
from util import load_sd

pytestmark = pytest.mark.gpu


def _glip(dev):
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
    from oracle import synth
    gen = synth.Gen(3031)
    sd = synth.detector_sd(gen, bias0=-1.0)
    ids, am, pmap = synth.prompt(13, 2, 256, gen)
    bank = synth.query_bank(pmap, 5, gen)
    model = GeneralizedVLRCNN_New(mq_glip_t_cfg())
    full = dict(sd)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            full[k] = v
    model = load_sd(model, full).to(dev).eval()
    model.query_selector.set_query_bank(bank)
    return model, {"input_ids": ids, "attention_mask": am}, pmap, synth.images(gen, 2, 160, 224), [(160, 224), (160, 224)]


def _gdino(dev):
    from test_gdino_asm_gpu import _build_model, _gdino_case
    sd, ids, am, pmap, bank, img = _gdino_case(3032, 2, 160, 224, 13, 2, 2, 100)
    model = _build_model(sd, 2, 2, 100, dev)
    model.query_selector.set_query_bank(bank)
    return model, {"input_ids": ids, "attention_mask": am}, pmap, img, [(160, 224), (138, 190)]


IDS, ORIG = [11, 4], [(240, 336), (207, 285)]


def _case(boxlists, labels):
    """GT at the original sizes from every second detection (jittered), the first one crowd; label -> json id = 3 * label + 1
    for the labels in ``labels`` except the largest."""
    l2c = {int(lab): 3 * int(lab) + 1 for lab in labels[:-1]}
    rng = np.random.default_rng(3)
    anns, images = [], []
    for b, bl in enumerate(boxlists):
        oh, ow = ORIG[b]
        w0, h0 = bl.size
        rx, ry = np.float32(ow / w0), np.float32(oh / h0)
        xyxy = bl.bbox.cpu().numpy() * np.array([rx, ry, rx, ry], np.float32)
        labs = bl.get_field("labels").cpu().numpy()
        for k in range(0, len(labs), 2):
            if int(labs[k]) not in l2c:
                continue
            x1, y1, x2, y2 = (xyxy[k] + rng.normal(0, 2, 4)).tolist()
            w, h = max(x2 - x1, 1.0), max(y2 - y1, 1.0)
            anns.append({"id": len(anns) + 1, "image_id": IDS[b], "category_id": l2c[int(labs[k])], "bbox": [x1, y1, w, h],
                         "area": w * h, "iscrowd": int(len(anns) == 0)})
        images.append({"id": IDS[b], "width": ow, "height": oh})
    gt = {"images": images, "annotations": anns,
          "categories": [{"id": c, "name": f"c{c}"} for c in sorted(set(l2c.values()))]}
    return gt, l2c


def _check(gt, l2c, packed, image_sizes, boxlists, dev):
    from mqdet_b200.engine.coco_eval import CocoEvaluator, CocoGroundTruth
    assert len(gt["annotations"]) > 3
    a = CocoEvaluator(CocoGroundTruth(gt, dev), label_to_category=l2c)
    a.update_packed(packed, IDS, image_sizes, ORIG)
    a.accumulate()
    b_ = CocoEvaluator(CocoGroundTruth(gt, dev), label_to_category=l2c)
    b_.update([(i, bl) for i, bl in zip(IDS, boxlists)])
    b_.accumulate()
    assert np.array_equal(a.eval["precision"], b_.eval["precision"]) and np.array_equal(a.eval["recall"], b_.eval["recall"])
    per = [(i, bl.bbox.cpu().numpy(), bl.size, bl.get_field("scores").cpu().numpy(), bl.get_field("labels").cpu().numpy())
           for i, bl in zip(IDS, boxlists)]
    o = co.evaluate(gt, co.prepare(gt, per, l2c))
    assert np.array_equal(a.eval["precision"], o.eval["precision"])
    assert np.array_equal(a.eval["recall"], o.eval["recall"])
    assert np.array_equal(a.summarize(), o.stats) and o.stats[0] > 0


@pytest.mark.parametrize("build", [_glip, _gdino], ids=["mq_glip_t", "mq_groundingdino_t"])
def test_update_packed_on_forward_device_output(build, dev):
    from mqdet_b200.structures.image_list import ImageList
    model, caps, pmap, img, sizes = build(dev)
    img[1, :, sizes[1][0]:, :] = 0
    img[1, :, :, sizes[1][1]:] = 0
    il = ImageList(img.to(dev), sizes)
    out = model.forward_device(il, caps, pmap)
    boxlists = model(il, captions=caps, positive_map=pmap)
    assert out["det_packed"].dim() == 3
    labels = sorted({int(v) for bl in boxlists for v in bl.get_field("labels").tolist()})
    assert len(labels) >= 3
    gt, l2c = _case(boxlists, labels)
    _check(gt, l2c, out["det_packed"], out["image_sizes"], boxlists, dev)


def test_update_packed_on_chunked_output(dev):
    """forward_chunked_device of a chunked MQ-GLIP: [G, B, max_out + 1, 6] with G = 3 chunks (27 classes)."""
    from mqdet_b200.structures.image_list import ImageList
    from test_lvis_eval_scale_gpu import _glip as chunked_glip
    model, chunks, img, sizes = chunked_glip(dev)
    il = ImageList(img.to(dev), sizes)
    caps = [{"input_ids": i, "attention_mask": a} for i, a, _ in chunks]
    pmaps = [pm for _, _, pm in chunks]
    out = model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=2)
    boxlists = model.forward_chunked(il, caps, pmaps, chunks_per_pass=2)
    assert out["det_packed"].shape[0] == 3
    labels = sorted({int(v) for bl in boxlists for v in bl.get_field("labels").tolist()})
    gt, l2c = _case(boxlists, labels)
    _check(gt, l2c, out["det_packed"], out["image_sizes"], boxlists, dev)
