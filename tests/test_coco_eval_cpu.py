"""CPU: tests/coco_eval_oracle.py (the restatement the GPU tests compare against).

1. Wrapper layer, pinned to the reference's own od_to_grounding/od_eval.py (do_od_evaluation -> prepare_for_coco_detection,
   evaluate_predictions_on_coco, summarize_per_category, COCOResults) run on the CPU with the reference's BoxList, over a
   stand-in ``pycocotools`` package whose COCO / COCOeval are the restatement's (pycocotools is not installed here and the
   reference does not ship it) and a stub ``Masker``.  The results json, the CSV text and the results dict must equal the
   restatement's.  Recorded under tests/golden/coco_eval_pins.pt (``MQDET_RECORD_PINS=1``) so it also runs without the reference.
2. The COCO-only rules on small hand-checked cases: crowd IoU and reuse, the maxDets 1 / 10 truncation per pair, false positives
   of a category absent from an image, zero-area detections, the GT id 0 rule, empty results.  These are not pinned to
   executable reference code (pycocotools is absent); they restate pycocotools' cocoeval.py / maskApi.c bbIou."""
import contextlib
import io
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

import coco_eval_oracle as co
from oracle import ref_loader
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "coco_eval_pins.pt")
_store = None


def pinned(name, fn):
    global _store
    if _store is None:
        _store = torch.load(PIN_FILE, weights_only=True) if os.path.exists(PIN_FILE) else {}
    if ref_loader.available():
        val = fn()
        if os.environ.get("MQDET_RECORD_PINS") == "1":
            _store[name] = val
            torch.save(_store, PIN_FILE)
        return val
    assert name in _store, f"{name}: no recorded result in {PIN_FILE}"
    return _store[name]


def _od_eval():
    """The reference's od_eval module, loaded over the stand-ins."""
    ref_loader.rpn_inference(lambda *a, **k: None)   # the reference's structures package (BoxList, boxlist_ops)
    if "mqdet_odref" in sys.modules:
        return sys.modules["mqdet_odref"], sys.modules["maskrcnn_benchmark.structures.bounding_box"].BoxList
    pc = types.ModuleType("pycocotools")
    pc.__path__ = []
    for sub, attrs in (("coco", {"COCO": co.COCO}), ("cocoeval", {"COCOeval": co.COCOeval})):
        m = types.ModuleType(f"pycocotools.{sub}")
        m.__dict__.update(attrs)
        sys.modules[f"pycocotools.{sub}"] = m
        setattr(pc, sub, m)
    sys.modules.setdefault("pycocotools", pc)
    for name in ("maskrcnn_benchmark.modeling", "maskrcnn_benchmark.modeling.roi_heads",
                 "maskrcnn_benchmark.modeling.roi_heads.mask_head", "maskrcnn_benchmark.modeling.roi_heads.mask_head.inference"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__path__ = []
            sys.modules[name] = m
    sys.modules["maskrcnn_benchmark.modeling.roi_heads.mask_head.inference"].Masker = object
    mod = ref_loader._load_file("mqdet_odref", "maskrcnn_benchmark/data/datasets/evaluation/od_to_grounding/od_eval.py")
    return mod, sys.modules["maskrcnn_benchmark.structures.bounding_box"].BoxList


def _run_reference(gt, updates, tmp_path):
    mod, BoxList = _od_eval()

    class Dataset:
        def __init__(self):
            self.coco = co.COCO(json.loads(json.dumps(gt)))
            self.id_to_img_map = {}
            self.contiguous_category_id_to_json_id = {c["id"]: c["id"] for c in gt["categories"]}

    ds = Dataset()
    preds = []
    for upd in updates:
        for img_id, box, in_size, score, cat in upd:
            bl = BoxList(torch.from_numpy(box), in_size, mode="xyxy")
            bl.add_field("scores", torch.from_numpy(score))
            bl.add_field("labels", torch.from_numpy(cat))
            ds.id_to_img_map[len(preds)] = img_id
            preds.append(bl)
    with contextlib.redirect_stdout(io.StringIO()):
        results, coco_results = mod.do_od_evaluation(ds, preds, box_only=False, output_folder=tmp_path, iou_types=("bbox",),
                                                     expected_results=(), expected_results_sigma_tol=4)
    with open(os.path.join(tmp_path, "bbox.csv")) as f:
        csv = f.read()
    return {"results_json": json.dumps(coco_results["bbox"]), "csv": csv,
            "results": {k: float(v) for k, v in results.results["bbox"].items()}}


@pytest.mark.parametrize("name", sorted(co.pin_cases()))
def test_wrapper_layer_matches_reference(name, tmp_path):
    gt, updates = co.pin_cases()[name]
    ref = pinned(f"coco_eval/{name}", lambda: _run_reference(gt, updates, str(tmp_path)))
    o, res = co.run_oracle(gt, updates, {c["id"]: c["id"] for c in gt["categories"]})
    assert json.dumps(res) == ref["results_json"], "prepare_for_coco_detection"
    names = {c["id"]: c["name"] for c in gt["categories"]}
    assert co.per_category_csv(o.eval["precision"], o.params.catIds, names) == ref["csv"]
    assert {k: float(v) for k, v in co.coco_results(o.stats)["bbox"].items()} == ref["results"]


# ---- the COCO-only rules, hand-checked --------------------------------------------------------------------------------------
def _gt(anns, n_img=1, cats=(1, 2)):
    return {"images": [{"id": i + 1, "width": 100, "height": 100} for i in range(n_img)],
            "categories": [{"id": c, "name": f"c{c}"} for c in cats], "annotations": anns}


def _ann(i, img, cat, box, crowd=0, area=None):
    return {"id": i, "image_id": img, "category_id": cat, "bbox": box, "area": box[2] * box[3] if area is None else area,
            "iscrowd": crowd}


def _det(img, cat, box, score):
    return {"image_id": img, "category_id": cat, "bbox": box, "score": score}


def test_crowd_iou_and_reuse():
    """A crowd GT: IoU = inter / detection area, never used up, ignored: two detections inside it are both ignored."""
    gt = _gt([_ann(1, 1, 1, [0, 0, 50, 50], crowd=1), _ann(2, 1, 1, [60, 60, 20, 20])])
    res = [_det(1, 1, [10, 10, 20, 20], 0.9), _det(1, 1, [12, 12, 20, 20], 0.8)]
    assert co.bb_iou([[10, 10, 20, 20]], [[0, 0, 50, 50]], [1])[0, 0] == 1.0
    ev = co.evaluate(gt, res)
    e = ev.pairs[1, 1][0]
    assert (e["dtMatches"] == 1).all() and e["dtIgnore"].all()
    assert (ev.eval["recall"][:, 0, 0, 2] == 0).all() and (ev.eval["precision"][:, :, 0, 0, 2] == 0).all()


def test_max_dets_truncation_per_pair():
    """maxDets 1 / 10 count only the first 1 / 10 detections of each (image, category) pair by score."""
    gt = _gt([_ann(1, 1, 1, [0, 0, 40, 40]), _ann(2, 1, 1, [50, 50, 40, 40])])
    res = [_det(1, 1, [0, 0, 40, 40], 0.5), _det(1, 1, [50, 50, 40, 40], 0.4)] + \
        [_det(1, 1, [1, 90, 5, 5], 0.3 - k / 100) for k in range(12)]
    ev = co.evaluate(gt, res)
    assert ev.eval["recall"][0, 0, 0].tolist() == [0.5, 1.0, 1.0]
    assert ev.eval["precision"][0, 0, 0, 0].tolist() == [1 / (1 + np.spacing(1)), 1.0, 1.0]   # tp / (tp + fp + eps)


def test_absent_category_gives_false_positives():
    """No federated filter: a detection of a category without a GT in its image is a false positive."""
    gt = _gt([_ann(1, 1, 1, [0, 0, 40, 40]), _ann(2, 2, 2, [0, 0, 40, 40])], n_img=2)
    res = [_det(1, 2, [0, 0, 40, 40], 0.9), _det(2, 2, [0, 0, 40, 40], 0.5)]
    ev = co.evaluate(gt, res)
    assert (1, 2) in ev.pairs
    assert ev.eval["recall"][0, 1, 0, 2] == 1.0
    assert ev.eval["precision"][0, 0, 1, 0, 2] == 0.5        # the best precision at recall 0 is 1 / 2


def test_zero_area_detection_is_kept():
    """No get_ann_ids area filter: a zero-area detection is evaluated (a false positive in the ranges holding area 0)."""
    gt = _gt([_ann(1, 1, 1, [0, 0, 40, 40])])
    ev = co.evaluate(gt, [_det(1, 1, [5, 5, 0, 10], 0.9), _det(1, 1, [0, 0, 40, 40], 0.5)])
    e = ev.pairs[1, 1]
    assert len(e[0]["dtScores"]) == 2
    assert not e[0]["dtIgnore"][0, 0] and not e[1]["dtIgnore"][0, 0]      # area 0 is inside "all" and "small"
    assert ev.eval["precision"][0, 0, 0, 0, 2] == 0.5


def test_gt_id_zero():
    """A match to the GT with id 0 uses it up but counts as unmatched: a false positive, ignored when its area is outside the
    range."""
    gt = _gt([_ann(0, 1, 1, [0, 0, 40, 40]), _ann(1, 1, 1, [50, 50, 40, 40])])
    ev = co.evaluate(gt, [_det(1, 1, [0, 0, 40, 40], 0.9), _det(1, 1, [1, 1, 40, 40], 0.8), _det(1, 1, [50, 50, 40, 40], 0.7)])
    e = ev.pairs[1, 1]
    assert e[0]["dtMatches"][0].tolist() == [0, 0, 1]
    assert not e[0]["dtIgnore"][0].any()
    assert e[3]["dtIgnore"][0].tolist() == [True, True, True]           # "large": every area (1600) is outside it
    assert ev.eval["recall"][0, 0, 0, 2] == 0.5


def test_empty_results():
    """No detections: zeros where the category has GTs, -1 elsewhere; the summary's means over entries > -1."""
    gt = _gt([_ann(1, 1, 1, [0, 0, 40, 40])])
    ev = co.evaluate(gt, [])
    assert (ev.eval["precision"][:, :, 0, 0] == 0).all() and (ev.eval["precision"][:, :, 1] == -1).all()
    assert (ev.eval["recall"][:, 0, 0] == 0).all() and (ev.eval["recall"][:, 1] == -1).all()
    assert ev.stats[0] == 0 and ev.stats[3] == -1


def test_unknown_image_raises_in_load_res():
    gt = _gt([_ann(1, 1, 1, [0, 0, 40, 40])])
    with pytest.raises(AssertionError, match="do not correspond"):
        co.evaluate(gt, [_det(7, 1, [0, 0, 40, 40], 0.9)])


# ---- the core, pinned to the reference's own LVISEval where the two protocols coincide -------------------------------------
def core_cases():
    """name -> (gt, updates): no crowd, GT ids >= 1, positive areas, <= 100 detections per (image, category) and <= 300 per
    image, only GT categories.  With every category without a GT in an image listed as negative there and nothing marked not
    exhaustive, LVIS standard AP (top 300 per image, federated filter, area filter) evaluates exactly what COCOeval does at
    maxDets 100."""
    g0 = co.synth_gt(21)
    g1 = co.synth_gt(22, n_img=8, n_cat=4, per_img=10)
    return {"core": (g0, co.synth_updates(g0, 31, pin=True)),
            "core_dense": (g1, co.synth_updates(g1, 32, n_upd=2, per_img=100, pin=True))}


def _lvis_format(gt):
    """The COCO-format case as an LVIS file: every category without a GT in an image is negative there."""
    present = {}
    for a in gt["annotations"]:
        present.setdefault(a["image_id"], set()).add(a["category_id"])
    cids = [c["id"] for c in gt["categories"]]
    return {"images": [dict(im, neg_category_ids=[c for c in cids if c not in present.get(im["id"], set())],
                            not_exhaustive_category_ids=[]) for im in gt["images"]],
            "categories": [dict(c, frequency="f") for c in gt["categories"]], "annotations": gt["annotations"]}


def _canonical(pairs):
    """Pair keys [P, 2] and the concatenated (matches, ignore) arrays of every area range, in key order."""
    keys = sorted(pairs)
    ints = [np.asarray(x, np.int64).ravel() for k in keys for e in pairs[k] for x in e]
    return np.array(keys, np.int64).reshape(-1, 2), np.concatenate(ints) if ints else np.zeros(0, np.int64)


def _run_lvis_eval(gt, results, tmp_path):
    import test_lvis_eval_cpu as tl
    mod, _ = tl._reference()
    path = os.path.join(tmp_path, "gt.json")
    with open(path, "w") as f:
        json.dump(_lvis_format(gt), f)
    with contextlib.redirect_stdout(io.StringIO()):
        lvis = mod.LVIS(path)
        le = mod.LVISEval(lvis, mod.LVISResults(lvis, json.loads(json.dumps(results)), max_dets=300), "bbox")
        le.evaluate()
        le.accumulate()
    A, I = len(le.params.area_rng), len(le.params.img_ids)
    pairs = {}
    for k, cat_id in enumerate(le.params.cat_ids):
        for a in range(A):
            for i, img_id in enumerate(le.params.img_ids):
                e = le.eval_imgs[k * A * I + a * I + i]
                if e is not None:
                    pairs.setdefault((img_id, cat_id), []).append((e["dt_matches"], e["dt_ignore"]))
    keys, ints = _canonical(pairs)
    return {"pair_keys": torch.from_numpy(keys), "match": tl._sha(ints), "precision": torch.from_numpy(le.eval["precision"]),
            "recall": torch.from_numpy(le.eval["recall"])}


@pytest.mark.parametrize("name", sorted(core_cases()))
def test_core_matches_reference_lvis_eval(name, tmp_path):
    """Matching, ties, stable-sort accumulation and the 101-point sampling of the restatement at maxDets 100 equal the reference's
    own LVISEval (standard AP) run on the CPU, on cases where the protocols coincide."""
    import test_lvis_eval_cpu as tl
    gt, updates = core_cases()[name]
    assert not any(a["iscrowd"] for a in gt["annotations"]) and min(a["id"] for a in gt["annotations"]) >= 1
    o, res = co.run_oracle(gt, updates)
    per_pair, per_img = {}, {}
    for r in res:
        per_pair[r["image_id"], r["category_id"]] = per_pair.get((r["image_id"], r["category_id"]), 0) + 1
        per_img[r["image_id"]] = per_img.get(r["image_id"], 0) + 1
        assert r["bbox"][2] * r["bbox"][3] > 0
    assert max(per_pair.values()) <= 100 and max(per_img.values()) <= 300 and max(per_pair.values()) > 10
    ref = pinned(f"coco_eval_core/{name}", lambda: _run_lvis_eval(gt, res, str(tmp_path)))
    keys, ints = _canonical({k: [(e["dtMatches"], e["dtIgnore"]) for e in v] for k, v in o.pairs.items()})
    assert np.array_equal(keys, ref["pair_keys"].numpy()), "evaluated (image, category) pairs"
    assert tl._sha(ints) == ref["match"], "per-(image, category) match / ignore arrays"
    assert np.array_equal(o.eval["precision"][..., 2], ref["precision"].numpy())
    assert np.array_equal(o.eval["recall"][..., 2], ref["recall"].numpy())
