"""CPU: test-time augmentation for MQ-GroundingDINO.

* tests/bbox_aug_gdino_oracle.py (packed detector rows -> transpose -> remove_boxes -> resize, then the merge) pinned to the
  reference's own maskrcnn_benchmark/data/datasets/evaluation/box_aug.py and BoxList, compiled from source as
  tests/test_bbox_aug_cpu.py does, on GroundingDINO-shaped passes (up to 900 rows in query order, boxes clipped at the border,
  empty passes, flipped passes).  Results are recorded under tests/golden/bbox_aug_gdino_pins.pt so that the comparison also runs
  where the reference is absent.
* The host logic of ``engine/bbox_aug`` for a ``GroundingDINO`` model over the ops test double (tests/hostlogic), in its own
  process.
"""
import os
import subprocess
import sys

import pytest
import torch

import bbox_aug_gdino_oracle as go
import bbox_aug_oracle as bo
import refpin
from oracle import ref_loader
from test_bbox_aug_cpu import _reference
from util import ROOT

PIN_FILE = os.path.join(ROOT, "tests", "golden", "bbox_aug_gdino_pins.pt")
_store = None
CASES = sorted(go.pin_cases())


def pinned(name, fn):
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


def _run_reference(c):
    """box_aug.py on the case: per pass the BoxList GroundingDINO returns (pass size, xyxy), transposed back when flipped,
    remove_boxes, resized to the original image, concatenated, merge_result_from_multi_scales."""
    ns = _reference(c["test"])
    BoxList = ns["BoxList"]
    parts = []
    for size, flip, rng, b, s, lab in c["passes"]:
        bl = BoxList(b.clone(), size, mode="xyxy")
        bl.add_field("labels", lab.clone())
        bl.add_field("scores", s.clone())
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
def test_packed_restatement_vs_reference_box_aug(name):
    c = go.pin_cases()[name]
    want = pinned(name, lambda: _run_reference(c))
    got = go.run_case(c)
    ub, us, ul = got["union"]
    assert torch.equal(ub, want["union_boxes"]) and torch.equal(us, want["union_scores"]) and torch.equal(ul, want["union_labels"])
    b, s, lab = got["result"]
    assert torch.equal(lab, want["labels"]) and torch.equal(s, want["scores"])
    if c["test"].SPECIAL_NMS == "vote" and c["test"].TH > 0:
        # numpy adds the scores of a cluster of eight or more pairwise; the restatement (and the kernel) add them in score order
        assert torch.allclose(b, want["boxes"], rtol=1e-5, atol=1e-4)
    else:
        assert torch.equal(b, want["boxes"])


def test_cases_cover_what_they_claim():
    cs = go.pin_cases()
    c = cs["two_scales_flip_nms"]
    assert [p[3].shape[0] for p in c["passes"]] == [900, 640, 0, 357] and c["M"] == 900
    u = go.run_case(c)["union"]
    assert 0 < u[0].shape[0] < 900 + 640 + 357                                  # the ranges dropped boxes
    first = c["passes"][0][3]
    assert [float((r[2] - r[0] + 1) * (r[3] - r[1] + 1)) for r in first[:2]] == [1024.0, 1056.0]   # lo^2 exactly: dropped
    for size, _, _, b, _, _ in c["passes"]:                                      # clipped at the border, as GroundingDINO's
        if b.shape[0]:
            assert (b[:, 0] == 0).any() and (b[:, 2] == size[0] - 1).any() and (b[:, 1] == 0).any() and (b[:, 3] == size[1] - 1).any()
    lens = [p[3].shape[0] for p in cs["unequal_ratios_nms"]["passes"]]
    assert lens == [1, 0, 300, 299]
    assert len(go.run_case(cs["unequal_ratios_nms"])["result"][1]) == 100        # the PRE_NMS_TOP_N cut engaged
    th0 = go.run_case(cs["two_scales_flip_th0"])
    assert th0["result"][0].shape[0] == th0["union"][0].shape[0]
    assert go.run_case(cs["all_empty"])["result"][0].shape[0] == 0
    for name in ("two_scales_flip_nms", "unequal_ratios_nms"):
        ub, _, ul = go.run_case(cs[name])["union"]
        assert bo.min_iou_margin(ub, ul, cs[name]["test"].TH) > 1e-6


def test_restated_collect_counts_overflow_and_bad_count_rows():
    g = torch.Generator().manual_seed(5)
    b, s, lab = go.gdino_rows(g, 40, (320, 240), 5)
    pk = torch.stack([go.pack(b, s, lab, 50), go.pack(b[:3], s[:3], lab[:3], 50)])
    pk[1, 50, 0] = 51.0
    m = go.collect_packed(go.empty_merged(2, 30), pk, (320, 240), (640, 480))
    assert m[0]["boxes"].shape[0] == 30 and m[0]["overflow"] == 10
    assert m[1]["boxes"].shape[0] == 0 and m[1]["overflow"] == go.BAD_COUNT


def test_groundingdino_cfg_has_the_tta_keys():
    """mq_groundingdino_t_cfg carries the TEST.* keys of config/defaults.py:856-867 that box_aug.py reads."""
    from mqdet_b200.config import mq_glip_t_cfg, mq_groundingdino_t_cfg
    t, ref = mq_groundingdino_t_cfg().TEST, mq_glip_t_cfg().TEST
    for k in ("USE_MULTISCALE", "SCALES", "RANGES", "MAX_SIZE", "FLIP", "SPECIAL_NMS", "TH", "PRE_NMS_TOP_N", "NUM_CLASSES",
              "SELECT_CLASSES"):
        assert getattr(t, k) == getattr(ref, k), k
    assert t.USE_MULTISCALE is False and t.MAX_SIZE == 2500 and t.FLIP is True and len(t.SCALES) == len(t.RANGES) == 12


def test_im_detect_bbox_aug_groundingdino_host_logic():
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostlogic", "bbox_aug_gdino_case.py")], capture_output=True,
                       text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "PASS bbox_aug_gdino" in r.stdout, (r.stdout[-1500:], r.stderr[-3000:])
