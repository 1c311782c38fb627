"""GPU: the device COCO box AP evaluator (mqdet_b200/engine/coco_eval.py on the kernels of csrc/lvis_eval.cu) against the numpy
restatement tests/coco_eval_oracle.py: per-(image, category, area range) match / ignore arrays identical, precision / recall fp64
arrays, stats, printed lines, results dict and per-category CSV identical, on the pinned cases and on a COCO-val-shaped set whose
pool is cut between updates.  Scores sit on a 1/64 grid and GT boxes are duplicated, so equal scores (broken by arrival, then
image id) and equal IoUs (a later GT replaces an earlier one) are exercised."""
import numpy as np
import pytest
import torch

import coco_eval_oracle as co
from mqdet_b200._lib import MqdetError
from mqdet_b200.engine.coco_eval import CocoEvaluator, CocoGroundTruth

pytestmark = pytest.mark.gpu


def _packed(upd, dev, gt):
    """One update as the detector's packed result [1, B, M + 1, 6] + ids and (h, w) sizes (the GT image's size as original)."""
    M = max(len(s) for *_, s, _ in upd)
    pk = torch.zeros((1, len(upd), M + 1, 6), dtype=torch.float32)
    wh = {im["id"]: (im["width"], im["height"]) for im in gt["images"]}
    for b, (_, box, _, score, cat) in enumerate(upd):
        n = len(score)
        pk[0, b, :n, :4] = torch.from_numpy(box)
        pk[0, b, :n, 4] = torch.from_numpy(score)
        pk[0, b, :n, 5] = torch.from_numpy(cat.astype(np.float32))
        pk[0, b, M, 0] = n
    ids = [u[0] for u in upd]
    in_hw = [(u[2][1], u[2][0]) for u in upd]
    orig_hw = [(wh.get(u[0], u[2])[1], wh.get(u[0], u[2])[0]) for u in upd]
    return pk.to(dev), ids, in_hw, orig_hw


def _run_device(gt, updates, dev, pool_rows=1 << 20):
    ev = CocoEvaluator(CocoGroundTruth(gt, dev), pool_rows=pool_rows)
    for upd in updates:
        ev.update_packed(*_packed(upd, dev, gt))
    ev.accumulate(want_match=True)
    return ev


def _device_pairs(ev):
    """{(image id, category id): per area range (dt matches [T, D], dt ignore [T, D], scores [D])} of the device result."""
    out = ev.last
    npair = int(out["n_paired"].item())
    order = out["order"][:npair].cpu().numpy()
    mg = out["match_gt"][:npair].cpu().numpy()
    tpb = out["tp_bits"][:npair].cpu().numpy().view(np.uint64)
    igb = out["ig_bits"][:npair].cpu().numpy().view(np.uint64)
    d = ev.detections()
    img, cat, score = d["image_id"][order], d["category_id"][order], d["score"][order]
    pairs, i = {}, 0
    while i < npair:
        j = i
        while j < npair and img[j] == img[i] and cat[j] == cat[i]:
            j += 1
        res = []
        for a in range(4):
            v = np.arange(a * 10, a * 10 + 10).astype(np.uint64)
            tp = ((tpb[i:j, None] >> v[None, :]) & np.uint64(1)).T.astype(bool)
            assert np.array_equal(tp, mg[i:j][:, a * 10:a * 10 + 10].T != 0)
            res.append((mg[i:j][:, a * 10:a * 10 + 10].T.astype(np.int64),
                        ((igb[i:j, None] >> v[None, :]) & np.uint64(1)).T.astype(bool), score[i:j].astype(np.float64)))
        pairs[int(img[i]), int(cat[i])] = res
        i = j
    return pairs


def _compare(ev, o, capsys=None):
    dp = _device_pairs(ev)
    op = {k: [(e["dtMatches"], e["dtIgnore"], e["dtScores"]) for e in v] for k, v in o.pairs.items() if len(v[0]["dtScores"])}
    assert sorted(dp) == sorted(op), "paired (image, category) keys"
    for k in op:
        for a in range(4):
            assert np.array_equal(dp[k][a][0], op[k][a][0]), (k, a, "matches")
            assert np.array_equal(dp[k][a][1], op[k][a][1]), (k, a, "ignore")
            assert np.array_equal(dp[k][a][2], op[k][a][2]), (k, a, "scores")
    assert ev.eval["precision"].shape == o.eval["precision"].shape
    assert np.array_equal(ev.eval["precision"], o.eval["precision"])
    assert np.array_equal(ev.eval["recall"], o.eval["recall"])
    stats = ev.summarize()
    assert np.array_equal(stats, o.stats)
    if capsys is not None:
        assert capsys.readouterr().out.splitlines() == o.lines
    assert ev.results() == co.coco_results(o.stats)


@pytest.mark.parametrize("name", sorted(co.pin_cases()))
def test_pinned_cases(name, dev, capsys, tmp_path):
    gt, updates = co.pin_cases()[name]
    ev = _run_device(gt, updates, dev)
    o, _ = co.run_oracle(gt, updates)
    capsys.readouterr()
    _compare(ev, o, capsys)
    text = ev.write_per_category_csv(str(tmp_path / "bbox.csv"))
    assert text == co.per_category_csv(o.eval["precision"], o.params.catIds, {c["id"]: c["name"] for c in gt["categories"]})
    assert open(tmp_path / "bbox.csv").read() == text


def test_reruns_bit_identical(dev):
    gt, updates = co.pin_cases()["crowd_id0"]
    a, b = _run_device(gt, updates, dev), _run_device(gt, updates, dev)
    assert a.eval["precision"].tobytes() == b.eval["precision"].tobytes()
    assert a.eval["recall"].tobytes() == b.eval["recall"].tobytes()
    for k in ("order", "tp_bits", "ig_bits", "match_gt"):
        assert torch.equal(a.last[k], b.last[k]), k


def coco_val_gt(seed, n_img=5000, n_cat=80, per_img=7):
    """COCO-val-shaped: 640 x 480 images, 80 categories (ids with gaps), ~36k GTs, ~1 % crowd, GT ids from 0, a duplicated GT
    in every tenth image."""
    rng = np.random.default_rng(seed)
    cats = [{"id": k + 1 + k // 10, "name": f"cat{k}"} for k in range(n_cat)]
    images, anns = [], []
    for i in range(n_img):
        images.append({"id": 10 * i + 3, "width": 640, "height": 480})
        present = rng.choice(n_cat, size=4, replace=False)
        for j in range(per_img + (i % 3 == 0)):
            w, h = rng.uniform(4, 300, 2)
            x, y = rng.uniform(0, 640 - w), rng.uniform(0, 480 - h)
            box = [float(x), float(y), float(w), float(h)]
            a = {"id": len(anns), "image_id": 10 * i + 3, "category_id": cats[int(present[j % 4])]["id"], "bbox": box,
                 "area": float(w * h * rng.uniform(0.5, 1.0)), "iscrowd": int(rng.random() < 0.01)}
            anns.append(a)
            if j == 0 and i % 10 == 0:
                anns.append(dict(a, id=len(anns), bbox=list(box)))
    return {"images": images, "annotations": anns, "categories": cats}


IN_HW, ORIG_HW = (800, 1066), (480, 640)


def coco_val_packed(gt, seed, image_ids, rows=100):
    """[1, B, rows + 1, 6] at a network size of 800 x 1066: 50 .. 100 detections per image, 60 % of them near a GT of the image
    (its category mostly), the rest anywhere, labels = category ids, scores on a 1/64 grid."""
    rng = np.random.default_rng(seed)
    cids = np.array([c["id"] for c in gt["categories"]])
    by_img = {}
    for a in gt["annotations"]:
        x, y, w, h = a["bbox"]
        by_img.setdefault(a["image_id"], []).append(([x, y, x + w, y + h], a["category_id"]))
    pk = np.zeros((1, len(image_ids), rows + 1, 6), np.float32)
    s = IN_HW[1] / ORIG_HW[1]
    for b, i in enumerate(image_ids):
        g = by_img[i]
        gb, gc = np.array([x[0] for x in g]), np.array([x[1] for x in g])
        xy = rng.uniform(0, 1, (rows, 2)) * [600.0, 440.0]
        box = np.concatenate([xy, xy + rng.uniform(4, 204, (rows, 2))], 1)
        lab = cids[rng.integers(0, len(cids), rows)]
        near = rng.random(rows) < 0.6
        k = rng.integers(0, len(gb), rows)
        box[near] = gb[k[near]] + rng.normal(0, 4, (int(near.sum()), 4))
        own = near & (rng.random(rows) < 0.8)
        lab[own] = gc[k[own]]
        pk[0, b, :rows, :4] = box * s
        pk[0, b, :rows, 4] = rng.integers(1, 64, rows) / 64.0
        pk[0, b, :rows, 5] = lab
        pk[0, b, rows, 0] = rng.integers(rows // 2, rows + 1)      # the slots past the count are empty
    return pk


def test_coco_val_shaped_set_with_cuts(dev, capsys):
    """5000 images, 80 categories, ~36k GTs with ~1 % crowd and ids from 0, 100 packed rows per image in updates of 250
    images; the pool holds the detections and two updates' rows, so it is cut (compacted) between updates."""
    gt = coco_val_gt(5)
    assert 30_000 < len(gt["annotations"]) < 42_000 and any(a["id"] == 0 for a in gt["annotations"])
    ids = [im["id"] for im in gt["images"]]
    parts = [ids[u * 250:(u + 1) * 250] for u in range(20)]
    pks = [coco_val_packed(gt, 100 + u, part) for u, part in enumerate(parts)]
    total = int(sum(pk[0, :, -1, 0].sum() for pk in pks))
    ev = CocoEvaluator(CocoGroundTruth(gt, dev), pool_rows=total + 2 * 250 * 100)
    cuts = []
    cut = ev._cut
    ev._cut = lambda: (cuts.append(ev.n), cut())[1]
    per = []
    for part, pk in zip(parts, pks):
        ev.update_packed(torch.from_numpy(pk).to(dev), part, [IN_HW] * len(part), [ORIG_HW] * len(part))
        for b, i in enumerate(part):
            n = int(pk[0, b, -1, 0])
            per.append((i, pk[0, b, :n, :4], (IN_HW[1], IN_HW[0]), pk[0, b, :n, 4], pk[0, b, :n, 5].astype(np.int64)))
    ev.accumulate(want_match=True)
    assert len(cuts) >= 2 and ev.n == total
    o = co.evaluate(gt, co.prepare(gt, per))
    capsys.readouterr()
    _compare(ev, o, capsys)
    assert o.stats[0] > 0.01


def test_update_with_boxlists_equals_update_packed(dev):
    """update() on the reference's input (BoxLists at the network size, resized to the GT image's size) = update_packed."""
    from mqdet_b200.structures.bounding_box import BoxList
    gt, updates = co.pin_cases()["basic"]
    a = _run_device(gt, updates, dev)
    ev = CocoEvaluator(CocoGroundTruth(gt, dev), pool_rows=1 << 20)
    for upd in updates:
        preds = []
        for img_id, box, in_size, score, cat in upd:
            bl = BoxList(torch.from_numpy(box).to(dev), in_size, mode="xyxy")
            bl.add_field("scores", torch.from_numpy(score).to(dev))
            bl.add_field("labels", torch.from_numpy(cat).to(dev))
            preds.append((img_id, bl))
        ev.update(preds)
    ev.accumulate()
    assert np.array_equal(ev.eval["precision"], a.eval["precision"])
    assert np.array_equal(ev.eval["recall"], a.eval["recall"])


def test_label_table_drops_unknown_labels(dev):
    """label_to_category as the reference's contiguous_category_id_to_json_id: labels 1..K, others dropped (also on images
    outside the GT file, which then do not raise)."""
    gt, updates = co.pin_cases()["basic"]
    l2c = {k + 1: c["id"] for k, c in enumerate(gt["categories"])}
    c2l = {v: k for k, v in l2c.items()}
    relabel = [[(i, b, s, sc, np.array([c2l.get(int(c), 77) for c in cat])) for i, b, s, sc, cat in upd] for upd in updates]
    relabel[0].append((424242, relabel[0][0][1], relabel[0][0][2], relabel[0][0][3], np.full(len(relabel[0][0][3]), 77)))
    ev = CocoEvaluator(CocoGroundTruth(gt, dev), label_to_category=l2c)
    for upd in relabel:
        ev.update_packed(*_packed(upd, dev, gt))
    ev.accumulate()
    o, _ = co.run_oracle(gt, relabel, l2c)
    assert np.array_equal(ev.eval["precision"], o.eval["precision"])
    assert np.array_equal(ev.eval["recall"], o.eval["recall"])


def test_empty_results(dev):
    gt, _ = co.pin_cases()["basic"]
    ev = CocoEvaluator(CocoGroundTruth(gt, dev))
    ev.accumulate()
    o = co.evaluate(gt, [])
    assert np.array_equal(ev.eval["precision"], o.eval["precision"])
    assert np.array_equal(ev.eval["recall"], o.eval["recall"])
    assert np.array_equal(ev.summarize(), o.stats)


def test_errors(dev):
    gt, updates = co.pin_cases()["basic"]
    pk, ids, s, o = _packed(updates[0], dev, gt)
    with pytest.raises(MqdetError, match="pool"):
        CocoEvaluator(CocoGroundTruth(gt, dev), pool_rows=pk.shape[1] * (pk.shape[2] - 1) - 1).update_packed(pk, ids, s, o)
    ev = CocoEvaluator(CocoGroundTruth(gt, dev))
    bad = pk.clone()
    bad[0, 0, -1, 0] = bad.shape[2]
    ev.update_packed(bad, ids, s, o)
    with pytest.raises(MqdetError, match="count row"):
        ev.accumulate()
    ev = CocoEvaluator(CocoGroundTruth(gt, dev))       # a detection on an image outside the GT file
    ev.update_packed(pk, [ids[0] + 1] + ids[1:], s, o)
    with pytest.raises(MqdetError, match="do not correspond"):
        ev.accumulate()
    ev = CocoEvaluator(CocoGroundTruth(gt, dev))       # an image outside the GT file without detections is accepted
    empty = pk.clone()
    empty[0, 0, -1, 0] = 0
    ev.update_packed(empty, [ids[0] + 1] + ids[1:], s, o)
    ev.accumulate()
