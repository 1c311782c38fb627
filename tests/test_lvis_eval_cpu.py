"""CPU: tests/lvis_eval_oracle.py (the restatement the GPU tests compare against) pinned to the reference's own
maskrcnn_benchmark/data/datasets/evaluation/lvis/lvis_eval.py (LvisEvaluatorFixedAP, LVISResults, LVISEval) and lvis.py (LVIS),
executed on the CPU, with the detections resized by the reference's own BoxList (engine/inference.py resize_box).

Stand-ins: ``pycocotools.mask.iou`` -> a fp64 bbIou written apart from the restatement (below); ``mdetr_dist`` -> a single
process.  The GT is synthetic and written to a temporary json.  Results are recorded under tests/golden/lvis_eval_pins.pt so
that the comparison also runs where the reference is absent."""
import contextlib
import hashlib
import importlib
import io
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

import lvis_eval_oracle as lo
from oracle import ref_loader
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "lvis_eval_pins.pt")
_store = None
CASES = sorted(lo.pin_cases())


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


def _sha(a):
    """Digest of an array's dtype, shape and bytes: the pins store it in place of the large exact arrays."""
    a = np.ascontiguousarray(a)
    return hashlib.sha256(str((a.dtype.str, a.shape)).encode() + a.tobytes()).hexdigest()


def coco_bb_iou(dt, gt, iscrowd):
    """pycocotools.mask.iou for lists of xywh boxes (maskApi.c bbIou), fp64, vectorised over the GTs."""
    if len(dt) == 0 or len(gt) == 0:
        return []
    d = np.asarray(dt, dtype=np.float64)
    g = np.asarray(gt, dtype=np.float64)
    out = np.zeros((len(d), len(g)))
    ga = g[:, 2] * g[:, 3]
    for i in range(len(d)):
        w = np.minimum(d[i, 2] + d[i, 0], g[:, 2] + g[:, 0]) - np.maximum(d[i, 0], g[:, 0])
        h = np.minimum(d[i, 3] + d[i, 1], g[:, 3] + g[:, 1]) - np.maximum(d[i, 1], g[:, 1])
        inter = w * h
        ok = (w > 0) & (h > 0)
        da = d[i, 2] * d[i, 3]
        out[i, ok] = inter[ok] / (da + ga[ok] - inter[ok])
    return out


def _reference():
    """(lvis_eval module, BoxList) of the reference, loaded with the two stand-ins."""
    ref_loader.rpn_inference(lambda *a, **k: None)   # installs the reference's structures package (BoxList)
    BoxList = sys.modules["maskrcnn_benchmark.structures.bounding_box"].BoxList
    if "mqdet_lvisref.lvis_eval" not in sys.modules:
        if "pycocotools" not in sys.modules:
            pc = types.ModuleType("pycocotools")
            pc.__path__ = []
            sys.modules["pycocotools"] = pc
        if "pycocotools.mask" not in sys.modules:
            m = types.ModuleType("pycocotools.mask")
            sys.modules["pycocotools.mask"] = m
            sys.modules["pycocotools"].mask = m
        sys.modules["pycocotools.mask"].iou = coco_bb_iou
        dist = types.ModuleType("maskrcnn_benchmark.utils.mdetr_dist")
        dist.all_gather = lambda x: [x]
        dist.is_main_process = lambda: True
        sys.modules["maskrcnn_benchmark.utils.mdetr_dist"] = dist
        sys.modules["maskrcnn_benchmark.utils"].mdetr_dist = dist
        pkg = types.ModuleType("mqdet_lvisref")
        pkg.__path__ = [os.path.join(ref_loader.REF, "maskrcnn_benchmark", "data", "datasets", "evaluation", "lvis")]
        sys.modules["mqdet_lvisref"] = pkg
        importlib.import_module("mqdet_lvisref.lvis_eval")
    return sys.modules["mqdet_lvisref.lvis_eval"], BoxList


def _run_reference(case, tmp_path):
    gt, updates, topk, fixed_ap = case
    mod, BoxList = _reference()
    path = os.path.join(tmp_path, "gt.json")
    with open(path, "w") as f:
        json.dump(gt, f)
    made = []

    class Recording(mod.LVISEval):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)

    with contextlib.redirect_stdout(io.StringIO()):
        lvis = mod.LVIS(path)
        ev = mod.LvisEvaluatorFixedAP(lvis, topk=topk, fixed_ap=fixed_ap)
        saved, mod.LVISEval = mod.LVISEval, Recording
        try:
            xywh = []
            for upd in updates:
                preds = []
                for img_id, box, in_size, orig_size, score, cat in upd:
                    bl = BoxList(torch.from_numpy(box), in_size, mode="xyxy").resize(orig_size)   # resize_box
                    preds.append((img_id, {"boxes": bl.bbox, "scores": torch.from_numpy(score),
                                           "labels": torch.from_numpy(cat)}))
                    xywh.append(mod.convert_to_xywh(bl.bbox).numpy())
                ev.update(preds)
            ev.synchronize_between_processes()
            strings = ev.summarize()
            if strings is None:   # _summarize_standard prints and returns nothing
                strings = made[-1].print_results()
        finally:
            mod.LVISEval = saved
    le = made[-1]
    A, I = len(le.params.area_rng), len(le.params.img_ids)
    pairs = {}
    for k, cat_id in enumerate(le.params.cat_ids):
        for a in range(A):
            for i, img_id in enumerate(le.params.img_ids):
                e = le.eval_imgs[k * A * I + a * I + i]
                if e is not None:
                    pairs.setdefault((img_id, cat_id), []).append(e)
    keys, ints, flts = lo.canonical(pairs)
    return {"xywh": _sha(np.concatenate(xywh)), "pair_keys": torch.from_numpy(keys), "match": _sha(ints),
            "dt_scores": _sha(flts), "precision": torch.from_numpy(le.eval["precision"]),
            "recall": torch.from_numpy(le.eval["recall"]),
            "results": torch.tensor([float(v) for v in le.results.values()], dtype=torch.float64),
            "result_keys": list(le.results.keys()), "strings": list(strings)}


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference(name, tmp_path):
    case = lo.pin_cases()[name]
    ref = pinned(f"lvis_eval/{name}", lambda: _run_reference(case, str(tmp_path)))
    gt, updates, topk, fixed_ap = case
    xywh = np.concatenate([lo.convert(b, s, os_) for upd in updates for _, b, s, os_, _, _ in upd])
    assert _sha(xywh) == ref["xywh"], "rule 1 conversion"
    o = lo.run_oracle(*case)
    keys, ints, flts = lo.canonical(o.pairs)
    assert np.array_equal(keys, ref["pair_keys"].numpy())
    assert _sha(ints) == ref["match"], "per-(image, category) match / ignore arrays"
    assert _sha(flts) == ref["dt_scores"]
    np.testing.assert_allclose(o.precision, ref["precision"].numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(o.recall, ref["recall"].numpy(), rtol=0, atol=1e-12)
    res, strings = o.summarize()
    assert list(res.keys()) == ref["result_keys"]
    np.testing.assert_allclose(np.array([float(v) for v in res.values()]), ref["results"].numpy(), rtol=0, atol=1e-12)
    assert strings == ref["strings"]


def test_cases_cover_the_rules():
    """The pinned cases hold what the rules turn on: > 10 000 detections of one category, a cut across updates, both protocols,
    ties in score, boundary areas, duplicates, an image and a category without GTs."""
    cases = lo.pin_cases()
    g, ups, topk, fixed = cases["fixed_big"]
    big = g["categories"][0]["id"]
    assert sum(int((c == big).sum()) for u in ups for *_, c in u) > 10000 and topk == 10000
    assert not cases["standard"][3] and any(len(s) > 300 for u in cases["standard"][1] for *_, s, _ in u)
    g0 = cases["fixed"][0]
    areas = [a["area"] for a in g0["annotations"]]
    assert 1024.0 in areas and 9216.0 in areas
    boxes = [tuple(a["bbox"]) + (a["image_id"], a["category_id"]) for a in g0["annotations"]]
    assert len(set(boxes)) < len(boxes)
    with_gt = {a["image_id"] for a in g0["annotations"]}
    assert any(im["id"] not in with_gt for im in g0["images"])
    assert any(c["id"] not in {a["category_id"] for a in g0["annotations"]} for c in g0["categories"])
    sc = np.concatenate([s for u in cases["fixed"][1] for *_, s, _ in u])
    assert len(np.unique(sc)) < len(sc)
