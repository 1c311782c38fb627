"""GPU: the LVIS evaluator at minival scale and on real detector output.

* A minival-shaped synthetic set (5000 images, 1203 categories, 50 000 GTs, 31 chunks x 100 packed rows per image = 15.5 M rows,
  updates of 500 images) against the numpy restatement: the fp64 precision / recall arrays and the summary identical.
* ``update_packed`` on ``forward_chunked_device`` of a small chunked MQ-GLIP and MQ-GroundingDINO model equals ``update`` on the
  BoxLists of ``forward_chunked`` resized to the original size (engine/inference.py resize_box), and the restatement."""
import numpy as np
import pytest
import torch

import lvis_eval_oracle as lo
from util import load_sd

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fixed_ap", [True, False])
def test_minival_shaped_set_equals_restatement(fixed_ap, dev):
    from mqdet_b200.engine.lvis_eval import LvisEvaluatorFixedAP, LvisGroundTruth
    gt = lo.minival_gt(5)
    ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, dev), fixed_ap=fixed_ap)
    o = lo.Oracle(gt, 10000, fixed_ap)
    ids = [im["id"] for im in gt["images"]]
    for u in range(10):
        part = ids[u * 500:(u + 1) * 500]
        pk = lo.minival_packed(gt, 100 + u, part)
        ev.update_packed(torch.from_numpy(pk).to(dev), part, [lo.MINIVAL_IN_HW] * len(part), [lo.MINIVAL_ORIG_HW] * len(part))
        o.update(lo.oracle_update_from_packed(pk, part, lo.MINIVAL_IN_HW, lo.MINIVAL_ORIG_HW))
    assert ev.n == 15_500_000
    ev.accumulate()
    o.evaluate()
    assert int(ev.last["n_paired"].item()) == len(o.dets_eval) > 10_000
    assert np.array_equal(ev.eval["precision"], o.precision)
    assert np.array_equal(ev.eval["recall"], o.recall)
    ev.summarize()
    r_o, _ = o.summarize()
    assert [float(v) for v in ev.results.values()] == [float(v) for v in r_o.values()]


def _chunks():
    from oracle import synth
    gen = synth.Gen(2077)
    chunks = synth.chunked_prompts(27, 10, 256, gen)
    bank = {}
    for _, _, pm in chunks:
        bank.update(synth.query_bank(pm, 5, gen))
    return gen, chunks, bank


def _glip(dev):
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.modeling.detector.generalized_vl_rcnn_new import GeneralizedVLRCNN_New
    from oracle import synth
    gen, chunks, bank = _chunks()
    sd = synth.detector_sd(gen, bias0=-1.0)
    model = GeneralizedVLRCNN_New(mq_glip_t_cfg(**{"MODEL.ATSS.DETECTIONS_PER_IMG": 300}))
    full = dict(sd)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            full[k] = v
    model = load_sd(model, full).to(dev).eval()
    model.query_selector.set_query_bank(bank)
    return model, chunks, synth.images(gen, 2, 160, 224), [(160, 224), (160, 224)]   # forward_flat: one size per batch


def _gdino(dev):
    from mqdet_b200.config import mq_groundingdino_t_cfg
    from mqdet_b200.modeling.groundingdino.groundingdino import GroundingDINO
    from oracle import synth
    gen, chunks, bank = _chunks()
    sd = synth.gdino_sd(gen, 2, 2, 100)
    cfg = mq_groundingdino_t_cfg(**{"GROUNDINGDINO.enc_layers": 2, "GROUNDINGDINO.dec_layers": 2, "GROUNDINGDINO.num_queries": 100,
                                    "MODEL.DYHEAD.NUM_CLASSES": 28})
    model = GroundingDINO(cfg)
    full = dict(sd)
    for k, v in model.state_dict().items():
        if k.endswith("relative_position_index"):
            full[k] = v
    model = load_sd(model, full).to(dev).eval()
    model.query_selector.set_query_bank(bank)
    return model, chunks, synth.rgb_images(gen, 2, 160, 224), [(160, 224), (138, 190)]


@pytest.mark.parametrize("build", [_glip, _gdino], ids=["mq_glip", "mq_groundingdino"])
def test_update_packed_on_chunked_model_output(build, dev):
    from mqdet_b200.engine.lvis_eval import LvisEvaluatorFixedAP, LvisGroundTruth
    from mqdet_b200.structures.image_list import ImageList
    model, chunks, img, sizes = build(dev)
    img[1, :, sizes[1][0]:, :] = 0
    img[1, :, :, sizes[1][1]:] = 0
    il = ImageList(img.to(dev), sizes)
    caps = [{"input_ids": i, "attention_mask": a} for i, a, _ in chunks]
    pmaps = [pm for _, _, pm in chunks]
    out = model.forward_chunked_device(il, caps, pmaps, chunks_per_pass=2)
    boxlists = model.forward_chunked(il, caps, pmaps, chunks_per_pass=2)
    ids, orig = [11, 4], [(240, 336), (207, 285)]
    # GT: jittered copies of a third of each image's detections (at the original size), so AP is not trivial
    rng = np.random.default_rng(3)
    anns, images = [], []
    for b, bl in enumerate(boxlists):
        oh, ow = orig[b]
        rx, ry = np.float32(ow / sizes[b][1]), np.float32(oh / sizes[b][0])
        xyxy = bl.bbox.numpy() * np.array([rx, ry, rx, ry], np.float32)
        labs = bl.get_field("labels").numpy()
        for k in range(0, len(labs), 2):
            x1, y1, x2, y2 = (xyxy[k] + rng.normal(0, 2, 4)).tolist()
            w, h = max(x2 - x1, 1.0), max(y2 - y1, 1.0)
            anns.append({"id": len(anns) + 1, "image_id": ids[b], "category_id": int(labs[k]), "bbox": [x1, y1, w, h],
                         "area": w * h, "iscrowd": 0})
        images.append({"id": ids[b], "width": ow, "height": oh, "neg_category_ids": [1, 2],
                       "not_exhaustive_category_ids": []})
    assert len(anns) > 3
    gt = {"images": images, "annotations": anns, "categories": [{"id": c, "frequency": "rcf"[c % 3]} for c in range(1, 28)]}
    a = LvisEvaluatorFixedAP(LvisGroundTruth(gt, dev))
    a.update_packed(out["det_packed"], ids, out["image_sizes"], orig)
    a.accumulate()
    b_ = LvisEvaluatorFixedAP(LvisGroundTruth(gt, dev))
    preds = []
    for b, bl in enumerate(boxlists):
        oh, ow = orig[b]
        rx, ry = np.float32(ow / sizes[b][1]), np.float32(oh / sizes[b][0])
        preds.append((ids[b], {"boxes": (bl.bbox * torch.tensor([rx, ry, rx, ry])).to(dev), "scores": bl.get_field("scores").to(dev),
                               "labels": bl.get_field("labels").to(dev)}))
    b_.update(preds)
    b_.accumulate()
    assert np.array_equal(a.eval["precision"], b_.eval["precision"]) and np.array_equal(a.eval["recall"], b_.eval["recall"])
    o = lo.Oracle(gt)
    o.update([(i, lo.convert(bl.bbox.numpy(), (s[1], s[0]), (og[1], og[0])), bl.get_field("scores").numpy(),
               bl.get_field("labels").numpy()) for i, bl, s, og in zip(ids, boxlists, sizes, orig)])
    o.evaluate()
    assert np.array_equal(a.eval["precision"], o.precision)
    assert a.summarize() == o.summarize()[1] and a.results["AP"] > 0
