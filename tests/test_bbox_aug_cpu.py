"""CPU: tests/bbox_aug_oracle.py (the restatement the GPU tests compare against) pinned to the reference's own
maskrcnn_benchmark/data/datasets/evaluation/box_aug.py, executed on the CPU.

The reference functions (remove_boxes, merge_result_from_multi_scales, boxlist_nms, bbox_vote) are compiled as they are from the
reference file and bound to the reference's own BoxList / cat_boxlist.  Stand-ins: ``layers.nms`` (a CUDA kernel) -> a CPU NMS
with the +1 box convention and the kernel's strict ``>``; ``Tensor.cuda()`` at the end of bbox_vote -> identity.  Results are
recorded under tests/golden/bbox_aug_pins.pt so that the comparison also runs where the reference is absent."""
import ast
import os
import sys
from types import SimpleNamespace as NS

import numpy as np
import pytest
import torch

import bbox_aug_oracle as bo
import refpin
from oracle import ref_loader
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "bbox_aug_pins.pt")
_store = None
CASES = sorted(bo.pin_cases())


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


def cpu_nms(boxes, scores, thresh):
    """csrc/cuda/nms.cu on the CPU: score-descending greedy suppression, IoU with +1 widths, strict '>', kept indices ascending.
    Written apart from the restatement (torch, box by box)."""
    order = torch.sort(scores, descending=True, stable=True)[1].tolist()
    b = boxes.float()
    area = (b[:, 2] - b[:, 0] + 1) * (b[:, 3] - b[:, 1] + 1)
    keep = []
    for i in order:
        ok = True
        for j in keep:
            w = (torch.min(b[i, 2], b[j, 2]) - torch.max(b[i, 0], b[j, 0]) + 1).clamp(min=0)
            h = (torch.min(b[i, 3], b[j, 3]) - torch.max(b[i, 1], b[j, 1]) + 1).clamp(min=0)
            inter = w * h
            if inter / (area[j] + area[i] - inter) > thresh:
                ok = False
                break
        if ok:
            keep.append(i)
    return torch.tensor(sorted(keep), dtype=torch.long)


def _reference(test_cfg):
    path = os.path.join(ref_loader.REF, "maskrcnn_benchmark", "data", "datasets", "evaluation", "box_aug.py")
    want = ("remove_boxes", "merge_result_from_multi_scales", "boxlist_nms", "bbox_vote")
    tree = ast.parse(open(path).read())
    fns = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in want]
    assert len(fns) == len(want)
    ref_loader.rpn_inference(lambda *a, **k: None)   # installs the reference's structures package
    ns = {"torch": torch, "np": np, "cfg": NS(TEST=test_cfg), "nms": cpu_nms, "soft_nms": None,
          "BoxList": sys.modules["maskrcnn_benchmark.structures.bounding_box"].BoxList,
          "cat_boxlist": sys.modules["maskrcnn_benchmark.structures.boxlist_ops"].cat_boxlist}
    exec(compile(ast.Module(body=fns, type_ignores=[]), path, "exec"), ns)
    return ns


def _run_reference(c):
    ns = _reference(c["test"])
    BoxList = ns["BoxList"]
    parts = []
    for size, flip, rng, b, s, l in c["passes"]:
        bl = BoxList(b.clone(), size, mode="xyxy")
        bl.add_field("scores", s.clone())
        bl.add_field("labels", l.clone())
        if flip:
            bl = bl.transpose(0)
        if rng is not None:
            bl = ns["remove_boxes"]([bl], *rng)[0]
        parts.append(bl.resize(c["orig_size"]))
    union = BoxList(torch.cat([p.bbox for p in parts]), parts[0].size, parts[0].mode)
    union.add_field("scores", torch.cat([p.get_field("scores") for p in parts]))
    union.add_field("labels", torch.cat([p.get_field("labels") for p in parts]))
    cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        r = ns["merge_result_from_multi_scales"]([union])[0]
    finally:
        torch.Tensor.cuda = cuda
    return {"union_boxes": union.bbox, "union_scores": union.get_field("scores"), "union_labels": union.get_field("labels"),
            "boxes": r.bbox.float(), "scores": r.get_field("scores").float(), "labels": r.get_field("labels")}


@pytest.mark.parametrize("name", CASES)
def test_restatement_vs_reference_box_aug(name):
    c = bo.pin_cases()[name]
    want = pinned(name, lambda: _run_reference(c))
    got = bo.run_case(c)
    ub, us, ul = got["union"]
    assert torch.equal(ub, want["union_boxes"]) and torch.equal(us, want["union_scores"]) and torch.equal(ul, want["union_labels"])
    b, s, l = got["result"]
    assert torch.equal(l, want["labels"]) and torch.equal(s, want["scores"]), (l, want["labels"])
    if c["test"].SPECIAL_NMS == "vote" and c["test"].TH > 0:
        # numpy adds the scores of a cluster of eight or more pairwise; the restatement (and the kernel) add them in score order
        assert torch.allclose(b, want["boxes"], rtol=1e-5, atol=1e-4)
    else:
        assert torch.equal(b, want["boxes"])
        if c["test"].TH > 0:
            assert bo.min_iou_margin(ub, ul, c["test"].TH) > 1e-6


def test_cases_cover_what_they_claim():
    cs = bo.pin_cases()
    u = bo.run_case(cs["equal_nms"])["union"]
    n_in = sum(p[3].shape[0] for p in cs["equal_nms"]["passes"])
    assert 0 < u[0].shape[0] < n_in                                   # the ranges dropped boxes
    areas = [(b[2] - b[0] + 1) * (b[3] - b[1] + 1) for b in cs["equal_nms"]["passes"][0][3][-4:]]
    assert [float(a) for a in areas[:2]] == [400.0, 40000.0]           # exactly on lo^2 / hi^2: dropped, their neighbours kept
    assert ((u[2] < 1) | (u[2] > 5)).any()                             # labels outside 1..NUM_CLASSES-1 reach the merge
    dup = (u[0] == torch.tensor([100., 50., 180., 140.])).all(1) & (u[1] == 0.77)
    assert int(dup.sum()) == 2                                         # a pass and a flipped pass found the same box
    r = bo.run_case(cs["topn_ties"])["result"]
    assert r[0].shape[0] == 9 and float(r[1].min()) == 0.5             # 6 asked, the five 0.5s tie at the cut
    assert bo.run_case(cs["empty"])["result"][0].shape[0] == 0
    lv = cs["unequal_vote"]
    assert int((torch.cat([p[5] for p in lv["passes"]]) == 5).sum()) == 1
    b, s, l, mem = bo.merge(*bo.run_case(lv)["union"], bo.class_list(lv["test"]), 0.6, "vote", 1000, want_members=True)
    assert max(len(m) for m in mem) >= 8 and int((l == 5).sum()) == 1
    assert set(bo.run_case(cs["select_classes"])["result"][2].tolist()) == {2, 4}


def test_unimplemented_modes_name_the_key():
    from mqdet_b200.config import mq_glip_t_cfg
    from mqdet_b200.engine import bbox_aug
    cfg = mq_glip_t_cfg()
    assert cfg.TEST.USE_MULTISCALE is False and len(cfg.TEST.SCALES) == len(cfg.TEST.RANGES) == 12
    for key in ("soft-nms", "soft-vote"):
        cfg.TEST.SPECIAL_NMS = key
        with pytest.raises(NotImplementedError, match=key):
            bbox_aug._mode(cfg.TEST)
    cfg.TEST.SELECT_CLASSES = (4, 2)
    with pytest.raises(ValueError, match="ascending"):
        bbox_aug._classes(cfg.TEST, "cpu")
