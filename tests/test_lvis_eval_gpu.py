"""GPU: the device LVIS evaluator (mqdet_b200/engine/lvis_eval.py, csrc/lvis_eval.cu) against the numpy restatement
tests/lvis_eval_oracle.py (itself pinned to the reference by tests/test_lvis_eval_cpu.py): per-(image, category) match / ignore
arrays identical, precision / recall fp64 arrays and the summary identical, on the pinned cases and on a larger set whose pool
is cut between updates.  Ties: scores sit on a 1/64 grid and GT boxes are duplicated, so equal scores (broken by arrival, then
image id) and equal IoUs (a later GT replaces an earlier one) are exercised; the device computes every IoU with the same IEEE
operations as the restatement, so thresholds compare identically."""
import numpy as np
import pytest
import torch

import lvis_eval_oracle as lo
from mqdet_b200._lib import MqdetError
from mqdet_b200.engine.lvis_eval import LvisEvaluatorFixedAP, LvisGroundTruth

pytestmark = pytest.mark.gpu


def _packed(upd, dev):
    """One update of a case as the detector's packed result [1, B, M + 1, 6] + ids and (h, w) sizes."""
    M = max(len(s) for *_, s, _ in upd)
    pk = torch.zeros((1, len(upd), M + 1, 6), dtype=torch.float32)
    for b, (_, box, _, _, score, cat) in enumerate(upd):
        n = len(score)
        pk[0, b, :n, :4] = torch.from_numpy(box)
        pk[0, b, :n, 4] = torch.from_numpy(score)
        pk[0, b, :n, 5] = torch.from_numpy(cat.astype(np.float32))
        pk[0, b, M, 0] = n
    ids = [u[0] for u in upd]
    in_hw = [(u[2][1], u[2][0]) for u in upd]
    orig_hw = [(u[3][1], u[3][0]) for u in upd]
    return pk.to(dev), ids, in_hw, orig_hw


def _run_device(gt, updates, topk, fixed_ap, dev, pool_rows=1 << 20):
    ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, dev), topk=topk, fixed_ap=fixed_ap, pool_rows=pool_rows)
    for upd in updates:
        ev.update_packed(*_packed(upd, dev))
    ev.accumulate(want_match=True)
    return ev


def _device_pairs(ev):
    """Dt-side canonical arrays of the device result: {(image id, category id): per area range dict}."""
    out = ev.last
    npair = int(out["n_paired"].item())
    order = out["order"][:npair].cpu().numpy()
    mg = out["match_gt"][:npair].cpu().numpy()
    igb = out["ig_bits"][:npair].cpu().numpy().view(np.uint64)
    d = ev.detections()
    img, cat, score = d["image_id"][order], d["category_id"][order], d["score"][order]
    pairs = {}
    i = 0
    while i < npair:
        j = i
        while j < npair and img[j] == img[i] and cat[j] == cat[i]:
            j += 1
        res = []
        for a in range(4):
            v = np.arange(a * 10, a * 10 + 10)
            res.append({"dt_matches": mg[i:j][:, v].T.astype(np.int64),
                        "dt_ignore": ((igb[i:j, None] >> v.astype(np.uint64)[None, :]) & np.uint64(1)).T.astype(np.int64),
                        "gt_ignore": np.zeros(0, np.int64), "gt_ids": np.zeros(0, np.int64),
                        "dt_scores": score[i:j].astype(np.float64)})
        pairs[int(img[i]), int(cat[i])] = res
        i = j
    return pairs


def _oracle_dt_pairs(o):
    return {k: [dict(e, gt_ignore=np.zeros(0, np.int64), gt_ids=np.zeros(0, np.int64),
                     dt_matches=np.asarray(e["dt_matches"], np.int64), dt_ignore=np.asarray(e["dt_ignore"], np.int64))
                for e in v] for k, v in o.pairs.items() if len(v[0]["dt_scores"])}


def _compare(ev, o):
    kd, idv, fd = lo.canonical(_device_pairs(ev))
    ko, ido, fo = lo.canonical(_oracle_dt_pairs(o))
    assert np.array_equal(kd, ko), "paired (image, category) keys"
    assert np.array_equal(idv, ido), "match / ignore arrays"
    assert np.array_equal(fd, fo), "detection order within pairs"
    assert np.array_equal(ev.eval["precision"], o.precision)
    assert np.array_equal(ev.eval["recall"], o.recall)
    strings = ev.summarize()
    r_o, s_o = o.summarize()
    assert list(ev.results) == list(r_o)
    assert all(ev.results[k] == r_o[k] for k in r_o)
    if ev.fixed_ap:
        assert strings == s_o


@pytest.mark.parametrize("name", sorted(lo.pin_cases()))
def test_pinned_cases(name, dev):
    gt, updates, topk, fixed_ap = lo.pin_cases()[name]
    _compare(_run_device(gt, updates, topk, fixed_ap, dev), lo.run_oracle(gt, updates, topk, fixed_ap))


@pytest.mark.parametrize("fixed_ap", [True, False])
def test_larger_set_with_cuts_between_updates(fixed_ap, dev):
    """250 images, 40 categories, 6 updates; a pool smaller than the arrivals forces cuts mid-stream (fixed AP: 3 updates'
    rows, with topk 700 biting; standard: room for 300 per image and one update)."""
    gt = lo.synth_gt(7, n_img=250, n_cat=40, per_img=8)
    updates = lo.synth_updates(gt, 8, n_upd=6, per_img=420)
    rows = max(len(u) * max(len(s) for *_, s, _ in u) for u in updates)
    total = sum(len(u) * max(len(s) for *_, s, _ in u) for u in updates)
    topk = 700 if fixed_ap else 10000
    pool = 3 * rows if fixed_ap else 300 * (len(gt["images"]) + 1) + rows
    assert pool < total
    ev = _run_device(gt, updates, topk, fixed_ap, dev, pool_rows=pool)
    _compare(ev, lo.run_oracle(gt, updates, topk, fixed_ap))


def test_reruns_bit_identical(dev):
    gt, updates, topk, fixed_ap = lo.pin_cases()["fixed_big"]
    a = _run_device(gt, updates, topk, fixed_ap, dev)
    b = _run_device(gt, updates, topk, fixed_ap, dev)
    assert a.eval["precision"].tobytes() == b.eval["precision"].tobytes()
    assert a.eval["recall"].tobytes() == b.eval["recall"].tobytes()
    for k in ("order", "tp_bits", "ig_bits", "match_gt"):
        assert torch.equal(a.last[k], b.last[k]), k


def test_update_with_boxlists_equals_update_packed(dev):
    """update() on the reference's input (xyxy at the original size) = update_packed on the network-size rows."""
    gt, updates, topk, fixed_ap = lo.pin_cases()["fixed"]
    a = _run_device(gt, updates, topk, fixed_ap, dev)
    ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, dev), topk=topk, fixed_ap=fixed_ap, pool_rows=1 << 20)
    for upd in updates:
        preds = []
        for img_id, box, in_size, orig_size, score, cat in upd:
            ratio = np.array([np.float32(orig_size[0] / in_size[0]), np.float32(orig_size[1] / in_size[1])] * 2, np.float32)
            preds.append((img_id, {"boxes": torch.from_numpy(box * ratio).to(dev), "scores": torch.from_numpy(score).to(dev),
                                   "labels": torch.from_numpy(cat).to(dev)}))
        ev.update(preds)
    ev.accumulate()
    assert np.array_equal(ev.eval["precision"], a.eval["precision"])
    assert np.array_equal(ev.eval["recall"], a.eval["recall"])


def test_full_pool_and_bad_count_raise(dev):
    gt, updates, topk, fixed_ap = lo.pin_cases()["fixed"]
    pk, ids, s, o = _packed(updates[0], dev)
    ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, dev), pool_rows=pk.shape[1] * (pk.shape[2] - 1) - 1)
    with pytest.raises(MqdetError, match="pool"):
        ev.update_packed(pk, ids, s, o)
    ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, dev), pool_rows=1 << 16)
    bad = pk.clone()
    bad[0, 0, -1, 0] = bad.shape[2]   # a count larger than the rows
    ev.update_packed(bad, ids, s, o)
    with pytest.raises(MqdetError, match="count row"):
        ev.accumulate()


def test_gt_ids_below_one_are_rejected(dev):
    gt = lo.synth_gt(3, n_img=2, n_cat=3, per_img=2)
    gt["annotations"][0]["id"] = 0
    with pytest.raises(ValueError, match=">= 1"):
        LvisGroundTruth(gt, dev)
