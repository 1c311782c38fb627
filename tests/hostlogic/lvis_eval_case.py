"""Host-logic dry run of ``engine/lvis_eval.py`` (CPU, throw-away process): ``LvisEvaluatorFixedAP`` composed over torch / numpy
stand-ins of ``ops.lvis_collect`` / ``ops.lvis_cut`` / ``ops.lvis_evaluate`` (each restating its kernel's specification in
include/mqdet_b200.h; the evaluation through tests/lvis_eval_oracle.py).  It checks the slot and arrival bookkeeping, the
(h, w) size convention, the cuts when the pool fills up, the label table, the errors and the summary — not the kernels.

    python tests/hostlogic/lvis_eval_case.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ops_double  # noqa: F401,E402  (patches mqdet_b200.ops; must come first)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import lvis_eval_oracle as lo  # noqa: E402
from mqdet_b200 import ops  # noqa: E402


def lvis_collect(pool, base, seq_base, packed, img_idx, ratios, cat_ids, *, label_map=None, need_img, bad):
    G, B, M1, _ = packed.shape
    M = M1 - 1
    if base + G * B * M > pool.cap:
        raise ops._lib.MqdetError("lvis_collect: pool full")
    cats = cat_ids.tolist()
    for b in range(B):
        for g in range(G):
            cnt = float(packed[g, b, M, 0])
            if not (0 <= cnt <= M and cnt == int(cnt)):
                bad += 1
            for r in range(M):
                slot = base + (b * G + g) * M + r
                pool.seq[slot] = seq_base + slot - base
                c, im = -1, int(img_idx[b])
                if r < cnt:
                    row = packed[g, b, r]
                    lab = int(row[5])
                    if label_map is not None:
                        lab = int(label_map[lab]) if 0 <= lab < label_map.numel() else -1
                    c = cats.index(lab) if lab in cats else -2
                    x1, y1, x2, y2 = (row[:4] * ratios[b].repeat(2)).tolist()
                    x1, y1, x2, y2 = [np.float32(v) for v in (x1, y1, x2, y2)]
                    pool.box[slot] = torch.tensor([x1, y1, x2 - x1, y2 - y1])
                    pool.score[slot] = row[4]
                if (not need_img and c == -2) or (need_img and im < 0):
                    c = -1
                pool.cat[slot], pool.img[slot] = c, im


def lvis_cut(src, n, dst, *, by_image, n_groups, k):
    cat, img = src.cat[:n].numpy(), src.img[:n].numpy()
    grp = img if by_image else cat
    ok = np.nonzero((cat != -1) & (grp >= 0))[0]
    o = ok[np.lexsort((src.seq[:n].numpy()[ok], -src.score[:n].numpy()[ok].astype(np.float64), grp[ok]))]
    keep = []
    for g in np.unique(grp[o]):
        keep += [i for i in o if grp[i] == g][:k]
    for f_src, f_dst in zip(src.fields(), dst.fields()):
        f_dst[:len(keep)] = f_src[keep]
    return torch.tensor([len(keep)], dtype=torch.int32)


def lvis_evaluate(pool, n, gt, *, want_match=False):
    d = lo.Detections()
    ok = np.nonzero(pool.cat[:n].numpy() >= 0)[0]
    img = pool.img[:n].numpy()[ok]
    d.img = np.where(img >= 0, gt.img_ids[np.maximum(img, 0)], -1)
    d.cat = gt.cat_ids[pool.cat[:n].numpy()[ok]]
    d.box, d.score, d.seq = pool.box[:n].numpy()[ok], pool.score[:n].numpy()[ok], pool.seq[:n].numpy()[ok]
    o = lo.Oracle(gt.dataset, topk=1 << 30, fixed_ap=True)
    o.dets = d
    o.evaluate()
    return {"precision": torch.from_numpy(o.precision), "recall": torch.from_numpy(o.recall),
            "n_paired": torch.tensor([len(o.dets_eval)], dtype=torch.int32)}


ops.lvis_collect, ops.lvis_cut, ops.lvis_evaluate = lvis_collect, lvis_cut, lvis_evaluate


def _packed(upd):
    M = max(len(s) for *_, s, _ in upd)
    pk = torch.zeros((1, len(upd), M + 1, 6))
    for b, (_, box, _, _, score, cat) in enumerate(upd):
        n = len(score)
        pk[0, b, :n, :4], pk[0, b, :n, 4], pk[0, b, :n, 5] = torch.from_numpy(box), torch.from_numpy(score), torch.from_numpy(cat)
        pk[0, b, M, 0] = n
    return pk, [u[0] for u in upd], [(u[2][1], u[2][0]) for u in upd], [(u[3][1], u[3][0]) for u in upd]


def main():
    from mqdet_b200._lib import MqdetError
    from mqdet_b200.engine.lvis_eval import LvisEvaluatorFixedAP, LvisGroundTruth
    gt = lo.synth_gt(1, n_img=6, n_cat=5, per_img=4)
    for fixed_ap, topk in ((True, 13), (False, 10000)):
        updates = lo.synth_updates(gt, 21, n_upd=3, per_img=400 if not fixed_ap else 30)
        rows = max(len(u) * max(len(s) for *_, s, _ in u) for u in updates)
        total = sum(len(u) * max(len(s) for *_, s, _ in u) for u in updates)
        ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, "cpu"), topk=topk, fixed_ap=fixed_ap,
                                  pool_rows=rows + topk * 5 if fixed_ap else total - 1)
        cuts = []
        cut = ev._cut
        ev._cut = lambda: (cuts.append(ev.n), cut())[1]
        for u in updates:
            ev.update_packed(*_packed(u))
        ev.accumulate()
        o = lo.run_oracle(gt, updates, topk, fixed_ap)
        assert len(cuts) >= 2, cuts                     # at least one cut while updating, one at accumulate
        assert np.array_equal(ev.eval["precision"], o.precision) and np.array_equal(ev.eval["recall"], o.recall)
        lines = ev.summarize()
        assert lines == (o.summarize()[1] if fixed_ap else None)
    # a label table: labels 0..4 name the categories in order
    ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, "cpu"), pool_rows=4096,
                              label_to_category=torch.tensor([c["id"] for c in gt["categories"]]))
    upd = lo.synth_updates(gt, 22, n_upd=1, per_img=20)[0]
    cat_pos = {c["id"]: k for k, c in enumerate(gt["categories"])}
    relabel = [(i, b, s, os_, sc, np.array([cat_pos.get(int(c), 99) for c in cat])) for i, b, s, os_, sc, cat in upd]
    ev.update_packed(*_packed(relabel))
    ev.accumulate()
    o = lo.run_oracle(gt, [upd], 10000, True)
    assert np.array_equal(ev.eval["precision"], o.precision)
    # a full pool and a bad count row
    pk = _packed(upd)
    try:
        LvisEvaluatorFixedAP(LvisGroundTruth(gt, "cpu"), pool_rows=pk[0].shape[1] * (pk[0].shape[2] - 1) - 1).update_packed(*pk)
        raise AssertionError("a full pool must raise")
    except MqdetError as e:
        assert "pool" in str(e)
    ev = LvisEvaluatorFixedAP(LvisGroundTruth(gt, "cpu"), pool_rows=4096)
    bad = pk[0].clone()
    bad[0, 0, -1, 0] = 0.5
    ev.update_packed(bad, *pk[1:])
    try:
        ev.accumulate()
        raise AssertionError("a bad count row must raise")
    except MqdetError as e:
        assert "count row" in str(e)
    print("PASS lvis_eval")


if __name__ == "__main__":
    main()
